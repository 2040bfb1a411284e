#!/usr/bin/env bash
# tools/brc_multi.sh N [brc-readcount arguments...] — one brc-readcount process per GPU, each computing its --shard of the
# regions (BAI-weighted, see brc_cli.cpp), STDOUT concatenated in rank order (ranks hold ascending site ranges).
# With --bgzf every rank writes a complete BGZF file; their concatenation is still one valid BGZF file, because each rank's
# closing EOF member is an ordinary empty member that readers step over (tests/test_bgzf_output.py checks it decompresses to the
# ranks' plain outputs concatenated).
set -euo pipefail
N=$1; shift
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
EXE="$HERE/../bam_readcount_b200/brc-readcount"
NDEV=${BRC_NDEV:-$N}
T="$(mktemp -d)"; trap 'rm -rf "$T"' EXIT
pids=()
for r in $(seq 0 $((N - 1))); do
  BRC_DEVICE=$((r % NDEV)) "$EXE" --shard "$r/$N" "$@" > "$T/out.$r" 2> "$T/err.$r" &
  pids+=($!)
done
rc=0
for p in "${pids[@]}"; do wait "$p" || rc=1; done
for r in $(seq 0 $((N - 1))); do cat "$T/out.$r"; done
cat "$T/err.0" >&2
exit $rc
