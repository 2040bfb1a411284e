#!/bin/bash
# tools/gpu_cli_timing.sh <tag> [blocks] — where the C++ host spends its time on a generated BAM (BRC_CLI_TIMING)
TAG=${1:-r02t}; NB=${2:-8000}; O=gpurun_out/$TAG; mkdir -p $O
mkdir -p /tmp/brc_txt
python - <<PY > $O/gen.log 2>&1
import sys, time, argparse
sys.path.insert(0, ".")
import bench
from bam_readcount_b200 import synth_cb
from oracle.oracle import REF_SAMTOOLS
spec = bench.make_spec("c4", argparse.Namespace(contigs=None, contig_blocks=None, c5_sites=None, c5_depth=None, c5_sites_per_window=None))
t = time.time(); info = synth_cb.write_sample_bam(spec, 0, 0, $NB, "/tmp/brc_txt", REF_SAMTOOLS); print(info, "written in %.1f s" % (time.time() - t))
PY
cat $O/gen.log
N=$(( NB * 1280 ))
( timeout 900 python -m pytest tests/test_cli.py tests/test_abi.py -m gpu -q -x 2>&1 | tail -5 ) > $O/pytest_cli.log 2>&1; tail -2 $O/pytest_cli.log
run() { name=$1; shift
  for rep in 1 2; do
    s=$(date +%s.%N)
    env "$@" BRC_CLI_TIMING=1 bam_readcount_b200/brc-readcount -w 0 -i -f /tmp/brc_txt/ref.fa /tmp/brc_txt/s.bam chr1:1-$N > /dev/null 2> $O/cli_${name}_$rep.err
    e=$(date +%s.%N); echo "$name rep $rep: wall $(python -c "print('%.3f' % ($e - $s))") s for $N bp"; grep "brc timing\] \(reference\|startup\|index\)" $O/cli_${name}_$rep.err
  done
}
run par X=1
run par_w4m BRC_CLI_WINDOW=4000000
run par_w2m BRC_CLI_WINDOW=2000000
s=$(date +%s.%N); bam_readcount_b200/brc-readcount -w 0 -i -f /tmp/brc_txt/ref.fa /tmp/brc_txt/s.bam chr1:1-$N 2>/dev/null | md5sum; e=$(date +%s.%N); echo "par to md5sum: $(python -c "print('%.3f' % ($e - $s))") s"
