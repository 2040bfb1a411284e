#!/bin/bash
# tools/gpu_session_gather.sh <tag> <n> — gather variants on the small sharded config + the e2e leg after the H2D reordering
TAG=${1:-r02g}; N=${2:-2}; O=gpurun_out/$TAG; mkdir -p $O
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29511"
S="bench.py --gpus $N --steps 3 --warmup 3 --contigs 4 --e2e-windows 0 --no-parity"
run() { name=$1; shift; env "$@" timeout 300 $TR $S > $O/g_$name.json 2> $O/g_$name.err; python - <<PY
import json
try:
    d=json.loads(open("$O/g_$name.json").read().strip().splitlines()[-1]); g=d["config"]["gather"]
    print("$name", "ms/step %.2f" % d["ms_per_step"], "without gather %.2f" % g["ms_per_step_without_gather"], "ok", g["verified_checksums"])
except Exception as ex:
    print("$name FAILED", ex, open("$O/g_$name.err").read()[-600:])
PY
}
run base X=1
run cemcpy NCCL_P2P_USE_CUDA_MEMCPY=1
run ch32 NCCL_MIN_NCHANNELS=32
run nthr256 NCCL_NTHREADS=256
run res64 BRC_K1_RESERVE_CTAS=64
# e2e leg (rank-local) after the H2D reordering
B="--config c3 --steps 3 --warmup 3 --no-cpu-baseline --no-e2e-text --no-parity"
e2e() { name=$1; shift; env "$@" timeout 300 python bench.py $B > $O/e2e_$name.json 2> $O/e2e_$name.err; echo "$name: $(python -c "import json;d=json.loads(open('$O/e2e_$name.json').read().strip().splitlines()[-1]);print('e2e %.2f ms h2d %d' % (d['e2e']['ms_per_step'], d['e2e']['h2d_bytes_per_step']))")"; }
e2e base X=1
e2e chunks4 BRC_PIPE_CHUNKS=4
e2e chunks16 BRC_PIPE_CHUNKS=16
e2e noelide BRC_NO_H2D_ELISION=1
( timeout 600 python -m pytest tests -m gpu -q -x 2>&1 | tail -4 ) > $O/pytest.log 2>&1; tail -2 $O/pytest.log
