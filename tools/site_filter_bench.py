"""Cost and payoff of the alternative-allele site filter (brc_set_site_filter); prints one JSON line.

Device: one C4-shaped window (12.5 Mb of a synthetic contig at 30x, 150 bp reads, -i), generated into HBM, run through the
device-resident path.  For each filter: the pileup kernel's and the selection's CUDA-event times (median of --runs after
--warmup), the fraction of printed sites kept and the bytes the results need on the host (dense packed records vs the compact
selection).  CLI: a synthetic BAM of --cli-mb Mb through brc-readcount with and without the filter: wall time and output bytes.

    python tools/site_filter_bench.py [--runs 10] [--warmup 3] [--cli-mb 4]
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

FILTERS = [None, (1, 0.0), (2, 0.0), (1, 0.2)]


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], text=True).strip()
    except Exception:
        pl = None
    return name, pl


def device_window(args):
    import torch
    from bam_readcount_b200 import stream as st
    from bam_readcount_b200 import synth_cb
    spec = synth_cb.Spec(seed=1234, mode=synth_cb.WGS, n_libs=8, contig_len=97656 * synth_cb.BLOCK_BP, n_contigs=1)
    w = st.wgs_windows(spec, 10)[0]
    device = torch.device("cuda", 0)
    max_reads = spec.window_reads(w.blk_lo, w.blk_hi) + 1024
    run = st.WindowRunner(spec, max_reads, device, dict(insertion_centric=True))
    # the reference characters on the host too, as a text-printing caller has them (the filter judges the printed reference base)
    run.eng.set_reference(w.contig, f"chr{w.contig + 1}", spec.contig_len, spec.ref_host(w.contig, 0, spec.contig_len), 0)
    run.cur_contig = w.contig
    out = {"window_sites": w.end - w.beg}
    try:
        for f in FILTERS:
            key = "off" if f is None else f"count{f[0]}_frac{f[1]}"
            if f is None:
                run.eng.clear_site_filter()
            else:
                run.eng.set_site_filter(*f)
            k1, sel = [], []
            for i in range(args.warmup + args.runs):
                run.launch(w, sec_cap=int((w.end - w.beg) * 0.2))
                run.done.synchronize()
                if i >= args.warmup:
                    k1.append(run.eng.stage_ms(1))
                    sel.append(run.eng.stage_ms(3))
            run.eng.fetch_device_results(run.stream.cuda_stream)
            r = dict(k1_ms=statistics.median(k1), launches=run.eng.launch_count())
            if f is None:
                pk = run.eng.packed()
                r["d2h_bytes"] = pk.nbytes()
                out["dense_d2h_bytes"] = pk.nbytes()
            else:
                s = run.eng.selected()
                r["select_ms"] = statistics.median(sel)
                r["kept_sites"] = int((s.emit == 1).sum())
                r["kept_fraction"] = r["kept_sites"] / (w.end - w.beg)
                r["shipped_sites"] = s.n_sites
                r["d2h_bytes"] = s.nbytes()
            out[key] = r
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
        base = [exe, "-w", "0", "-i", "-f", info["fasta"], info["bam"], region]
        for key, extra in (("off", []), ("count2", ["--min-alt-count", "2"]), ("frac0.2", ["--min-alt-fraction", "0.2"])):
            walls, nbytes = [], 0
            for _ in range(3):
                t0 = time.perf_counter()
                p = subprocess.run(base[:1] + extra + base[1:], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
                walls.append(time.perf_counter() - t0)
                assert p.returncode == 0
                nbytes = len(p.stdout)
            out[key] = dict(wall_s=statistics.median(walls), output_bytes=nbytes, lines=p.stdout.count(b"\n"))
        out["region_bp"] = nblk * synth_cb.BLOCK_BP - 1000
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cli-mb", type=float, default=4.0)
    args = ap.parse_args()
    name, pl = card()
    res = dict(card=name, power_limit_w=pl, device=device_window(args), cli=cli_runs(args))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
