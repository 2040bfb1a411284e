#!/bin/bash
# tools/gpu_session.sh <tag> — one visit to a GPU box: parity tests, the bench arms, kernel variants, ncu captures.
# Everything lands in gpurun_out/<tag>/ ; every step has its own timeout so a hang cannot eat the visit.
TAG=${1:-r02}
O=gpurun_out/$TAG
mkdir -p $O
nvidia-smi -L > $O/gpus.txt 2>&1
nproc > $O/host.txt; cat /sys/fs/cgroup/cpu.max >> $O/host.txt 2>&1; lscpu | head -20 >> $O/host.txt 2>&1
( timeout 900 python -m pytest tests -m gpu -q 2>&1 | tail -25 ) > $O/pytest.log 2>&1
echo "pytest done: $(tail -1 $O/pytest.log)"
B="--e2e-windows 0 --no-cpu-baseline --no-e2e-text --no-parity"
timeout 300 python bench.py --config c3 --steps 30 --warmup 3 $B > $O/bench_c3_main.json 2> $O/bench_c3_main.err
for v in bam_readcount_b200/variants/*.so; do
  n=$(basename $v .so)
  BRC_ENGINE_LIB=$PWD/$v timeout 300 python bench.py --config c3 --steps 30 --warmup 3 $B > $O/bench_c3_$n.json 2> $O/bench_c3_$n.err
done
python - <<PY
import json,glob
for f in sorted(glob.glob("$O/bench_c3_*.json")):
    try:
        d=json.loads(open(f).read().strip().splitlines()[-1]); r=d["roofline"]
        print(f.split("bench_c3_")[1], "ms/step %.3f k0 %.3f k1 %.3f frac %.3f gen %.3f" % (d["ms_per_step"], r["k0_ms"], r["k1_ms"], r["frac"], d["config"]["gen_ms_per_window"]))
    except Exception as ex:
        print(f, "FAILED", ex)
PY
timeout 600 python bench.py --config c3 --steps 20 --warmup 3 > $O/bench_c3_full.json 2> $O/bench_c3_full.err
echo "c3 full rc=$?"
timeout 900 python bench.py --steps 5 --warmup 3 > $O/bench_c4.json 2> $O/bench_c4.err
echo "c4 rc=$?"; tail -c 600 $O/bench_c4.err
timeout 600 python bench.py --steps 3 --warmup 3 --no-resident $B > $O/bench_c4_noresident.json 2> $O/bench_c4_noresident.err
timeout 600 python bench.py --config c5 --steps 2 --warmup 3 > $O/bench_c5.json 2> $O/bench_c5.err
echo "c5 rc=$?"; tail -c 400 $O/bench_c5.err
timeout 300 python bench.py --impl reference --steps 3 --warmup 1 > $O/bench_ref_c4.json 2> $O/bench_ref_c4.err
python - <<PY
import json
for f in ("bench_c3_full","bench_c4","bench_c4_noresident","bench_c5","bench_ref_c4"):
    try:
        d=json.loads(open("$O/"+f+".json").read().strip().splitlines()[-1])
        print(f, "value %.4g ms/step %.3f" % (d["value"], d["ms_per_step"]), "e2e", d.get("e2e",{}).get("ms_per_step"), "parity", d.get("parity",{}).get("identical"), "text", d.get("e2e_text",{}).get("value"), d.get("e2e_text",{}).get("compressed_span",{}).get("ms"))
    except Exception as ex:
        print(f, "FAILED", ex)
PY
# ncu: launch list of the bench command + one full capture of K1 and K0 on the C3 window
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -c 150 --csv --log-file $O/launches_c4.csv python bench.py --steps 1 --warmup 3 --contigs 1 $B > $O/bench_under_ncu_c4.log 2>&1
timeout 600 ncu --set full --clock-control none --import-source on -k regex:pileup_kernel -s 4 -c 1 -o $O/prof_k1 -f python bench.py --config c3 --steps 2 --warmup 3 $B > $O/ncu_k1.log 2>&1
timeout 600 ncu --set full --clock-control none --import-source on -k regex:read_precompute -s 4 -c 1 -o $O/prof_k0 -f python bench.py --config c3 --steps 2 --warmup 3 $B > $O/ncu_k0.log 2>&1
timeout 600 ncu --set full --clock-control none --import-source on -k regex:deep_site -s 4 -c 1 -o $O/prof_deep -f python bench.py --config c5 --steps 1 --warmup 3 --c5-sites 600 --no-parity > $O/ncu_deep.log 2>&1
timeout 600 ncu --set full --clock-control none --import-source on -k regex:bgzf_inflate -c 1 -o $O/prof_inflate -f python -m pytest tests/test_bgzf_device.py -q -m gpu -k span_equals > $O/ncu_inflate.log 2>&1
ls -la $O | tail -40
