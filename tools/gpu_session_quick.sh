#!/bin/bash
# tools/gpu_session_quick.sh <tag> — a short visit: parity tests, K1 variants on C3, C5, PCIe probe, one K1 capture.
TAG=${1:-r02q}
O=gpurun_out/$TAG
mkdir -p $O
( timeout 900 python -m pytest tests -m gpu -q 2>&1 | tail -25 ) > $O/pytest.log 2>&1
echo "pytest done: $(tail -1 $O/pytest.log)"
B="--e2e-windows 0 --no-cpu-baseline --no-e2e-text --no-parity"
timeout 300 python bench.py --config c3 --steps 30 --warmup 3 $B > $O/bench_c3_main.json 2> $O/bench_c3_main.err
for v in bam_readcount_b200/variants/*.so; do
  n=$(basename $v .so)
  BRC_ENGINE_LIB=$PWD/$v timeout 300 python bench.py --config c3 --steps 30 --warmup 3 $B > $O/bench_c3_$n.json 2> $O/bench_c3_$n.err
done
timeout 600 python bench.py --config c5 --steps 3 --warmup 3 > $O/bench_c5.json 2> $O/bench_c5.err
echo "c5 rc=$?"; tail -c 400 $O/bench_c5.err
timeout 600 python bench.py --config c3 --steps 10 --warmup 3 --no-cpu-baseline > $O/bench_c3_full.json 2> $O/bench_c3_full.err
timeout 300 python tools/pcie_numa_probe.py > $O/pcie_probe.txt 2>&1
python - <<PY
import json,glob
for f in sorted(glob.glob("$O/bench_*.json")):
    try:
        d=json.loads(open(f).read().strip().splitlines()[-1]); r=d["roofline"]
        print(f.split("/")[-1], "value %.4g ms/step %.3f k0 %.3f k1 %.3f frac %.3f" % (d["value"], d["ms_per_step"], r["k0_ms"], r["k1_ms"], r["frac"]), "e2e", d.get("e2e",{}).get("ms_per_step"), "span", d.get("e2e_text",{}).get("compressed_span",{}).get("ms"))
    except Exception as ex:
        print(f, "FAILED", ex)
PY
cat $O/pcie_probe.txt | tail -12
timeout 600 ncu --set full --clock-control none --import-source on -k regex:pileup_kernel -s 4 -c 1 -o $O/prof_k1 -f python bench.py --config c3 --steps 2 --warmup 3 $B > $O/ncu_k1.log 2>&1
timeout 600 ncu --set full --clock-control none --import-source on -k regex:bgzf_inflate -c 1 -o $O/prof_inflate -f python -m pytest tests/test_bgzf_device.py -q -m gpu -k span_equals > $O/ncu_inflate.log 2>&1
ls $O
