"""Cost and payoff of the site filter's entry bounds (brc_set_site_filter_bounds, --alt-min / --alt-max); prints one JSON line.

Device: the C4-shaped window of tools/site_filter_bench.py (12.5 Mb of a synthetic contig at 30x, 150 bp reads, -i) through the
device-resident path, for --min-alt-count 1 alone, --min-alt-count 2, and the fpfilter-like set below: the selection's
CUDA-event time (brc_last_stage_ms(3), median of --runs after --warmup), the sites kept and the bytes shipped to the host.
CLI: a synthetic BAM of --cli-mb Mb through brc-readcount with the same three filters: wall time and STDOUT bytes.

    python tools/site_filter_bounds_bench.py [--runs 10] [--warmup 3] [--cli-mb 4]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from site_filter_bench import card  # noqa: E402

# an alternative allele seen on both strands, at base quality >= 20, away from the read start
FPFILTER = {"num_plus_strand": ("1", None), "num_minus_strand": ("1", None), "avg_basequality": ("20", None),
            "avg_pos_as_fraction": ("0.10", None)}
FILTERS = {"count1": (1, None), "count2": (2, None), "fpfilter": (1, FPFILTER)}


def cli_flags(bounds):
    out = []
    for name, (lo, hi) in (bounds or {}).items():
        out += (["--alt-min", f"{name}={lo}"] if lo is not None else []) + (["--alt-max", f"{name}={hi}"] if hi is not None else [])
    return out


def device_window(args):
    import torch
    from bam_readcount_b200 import stream as st
    from bam_readcount_b200 import synth_cb
    spec = synth_cb.Spec(seed=1234, mode=synth_cb.WGS, n_libs=8, contig_len=97656 * synth_cb.BLOCK_BP, n_contigs=1)
    w = st.wgs_windows(spec, 10)[0]
    device = torch.device("cuda", 0)
    max_reads = spec.window_reads(w.blk_lo, w.blk_hi) + 1024
    run = st.WindowRunner(spec, max_reads, device, dict(insertion_centric=True))
    run.eng.set_reference(w.contig, f"chr{w.contig + 1}", spec.contig_len, spec.ref_host(w.contig, 0, spec.contig_len), 0)
    run.cur_contig = w.contig
    out = {"window_sites": w.end - w.beg}
    try:
        for key, (count, bounds) in FILTERS.items():
            run.eng.set_site_filter(count, 0.0, bounds=bounds)
            sel = []
            for i in range(args.warmup + args.runs):
                run.launch(w, sec_cap=int((w.end - w.beg) * 0.2))
                run.done.synchronize()
                if i >= args.warmup:
                    sel.append(run.eng.stage_ms(3))
            run.eng.fetch_device_results(run.stream.cuda_stream)
            s = run.eng.selected()
            kept = int((s.emit == 1).sum())
            out[key] = dict(select_ms=statistics.median(sel), select_ms_min=min(sel), select_ms_max=max(sel), kept_sites=kept,
                            kept_fraction=kept / (w.end - w.beg), shipped_sites=s.n_sites, d2h_bytes=s.nbytes(),
                            launches=run.eng.launch_count())
    finally:
        run.eng.close()
    return out


def cli_runs(args):
    from bam_readcount_b200 import build, synth_cb
    from oracle.oracle import REF_SAMTOOLS
    if not os.path.exists(REF_SAMTOOLS):
        return {"skipped": "oracle/_ref/samtools not built"}
    exe = build.build_cli()
    nblk = int(args.cli_mb * 1e6) // synth_cb.BLOCK_BP
    spec = synth_cb.Spec(seed=77, mode=synth_cb.WGS, n_libs=8, contig_len=(nblk + 4) * synth_cb.BLOCK_BP)
    out = {}
    with tempfile.TemporaryDirectory() as wd:
        info = synth_cb.write_sample_bam(spec, 0, 0, nblk, wd, REF_SAMTOOLS)
        region = f"chr1:1001-{nblk * synth_cb.BLOCK_BP}"
        base = ["-w", "0", "-i", "-f", info["fasta"], info["bam"], region]
        for key, (count, bounds) in FILTERS.items():
            walls, nbytes, lines = [], 0, 0
            for _ in range(3):
                t0 = time.perf_counter()
                p = subprocess.run([exe, "--min-alt-count", str(count)] + cli_flags(bounds) + base, stdout=subprocess.PIPE,
                                   stderr=subprocess.DEVNULL)
                walls.append(time.perf_counter() - t0)
                assert p.returncode == 0
                nbytes, lines = len(p.stdout), p.stdout.count(b"\n")
            out[key] = dict(wall_s=statistics.median(walls), stdout_bytes=nbytes, lines=lines)
        out["region_bp"] = nblk * synth_cb.BLOCK_BP - 1000
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cli-mb", type=float, default=4.0)
    args = ap.parse_args()
    name, pl = card()
    print(json.dumps(dict(card=name, power_limit_w=pl, device=device_window(args), cli=cli_runs(args))))


if __name__ == "__main__":
    main()
