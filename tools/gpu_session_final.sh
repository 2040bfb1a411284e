#!/bin/bash
# tools/gpu_session_final.sh <tag> — one 1-GPU visit: parity tests, the driver's own bench commands (timed by wall clock), ncu captures.
TAG=${1:-r02f}; O=gpurun_out/$TAG; mkdir -p $O
nvidia-smi -L > $O/gpus.txt 2>&1
nproc > $O/host.txt; cat /sys/fs/cgroup/cpu.max >> $O/host.txt 2>&1; lscpu | head -20 >> $O/host.txt 2>&1
t0=$(date +%s)
( timeout 900 python -m pytest tests -m gpu -q 2>&1 | tail -25 ) > $O/pytest.log 2>&1
echo "pytest done in $(( $(date +%s) - t0 )) s: $(tail -1 $O/pytest.log)"
t0=$(date +%s); timeout 300 python -c "import __graft_entry__ as g; g.smoke(); print('smoke ok')" > $O/smoke.log 2>&1; echo "smoke rc=$? in $(( $(date +%s) - t0 )) s: $(tail -1 $O/smoke.log)"
t0=$(date +%s); timeout 900 python bench.py > $O/bench_c4.json 2> $O/bench_c4.err; echo "bench.py (defaults) rc=$? in $(( $(date +%s) - t0 )) s"; tail -c 400 $O/bench_c4.err
t0=$(date +%s); timeout 600 python bench.py --impl reference > $O/bench_ref_c4.json 2> $O/bench_ref_c4.err; echo "bench.py --impl reference rc=$? in $(( $(date +%s) - t0 )) s"
t0=$(date +%s); timeout 600 python bench.py --config c3 --steps 20 --warmup 3 > $O/bench_c3_full.json 2> $O/bench_c3_full.err; echo "c3 rc=$? in $(( $(date +%s) - t0 )) s"
t0=$(date +%s); timeout 600 python bench.py --config c5 --steps 2 --warmup 3 > $O/bench_c5.json 2> $O/bench_c5.err; echo "c5 rc=$? in $(( $(date +%s) - t0 )) s"
python - <<PY
import json
for f in ("bench_c4","bench_ref_c4","bench_c3_full","bench_c5"):
    try:
        d=json.loads(open("$O/"+f+".json").read().strip().splitlines()[-1]); r=d.get("roofline") or {}
        print(f, "value %.4g ms/step %.3f" % (d["value"], d["ms_per_step"]), "frac", r.get("frac"), "k1", r.get("k1_ms"), "e2e", d.get("e2e",{}).get("ms_per_step"), d.get("e2e",{}).get("value"), "parity", d.get("parity",{}).get("identical"),
              "text", (d.get("e2e_text") or {}).get("value"), "cpu", (d.get("cpu_baseline") or {}).get("value"), (d.get("cpu_baseline") or {}).get("cores"), "clocks", d.get("clocks"))
    except Exception as ex:
        print(f, "FAILED", ex)
PY
[ -n "$SKIP_NCU" ] && { ls -la $O | tail -20; exit 0; }
B="--e2e-windows 0 --no-cpu-baseline --no-e2e-text --no-parity"
# ncu: launch list of the bench command + one full capture of K1, K0 and the deep kernel
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -c 150 --csv --log-file $O/launches_c4.csv python bench.py --steps 1 --warmup 3 --contigs 1 $B > $O/bench_under_ncu_c4.log 2>&1
timeout 600 ncu --set full --clock-control none --import-source on -k regex:pileup_kernel -s 4 -c 1 -o $O/prof_k1 -f python bench.py --config c3 --steps 2 --warmup 3 $B > $O/ncu_k1.log 2>&1
timeout 600 ncu --set full --clock-control none --import-source on -k regex:read_precompute -s 4 -c 1 -o $O/prof_k0 -f python bench.py --config c3 --steps 2 --warmup 3 $B > $O/ncu_k0.log 2>&1
timeout 600 ncu --set full --clock-control none --import-source on -k regex:deep_site -s 4 -c 1 -o $O/prof_deep -f python bench.py --config c5 --steps 1 --warmup 3 --c5-sites 600 --no-parity --no-cpu-baseline > $O/ncu_deep.log 2>&1
ls -la $O | tail -30
