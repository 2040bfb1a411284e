"""Time of the complex-record kernel (brc_set_complex_queries, stage 5) on two workloads, and of `--vcf --vcf-complex`
against plain `--vcf` where samtools is at hand to index the BAM.  Prints one JSON line with the card's name and power limit.

  wgs    tools/vcf_bench.py's input, a synthetic 2 Mb contig at 30x, with one complex record every 20 bp (REF 1-20 bp, two ALTs
         cut from a spanning read's bases and one no read carries), pushed as one region through brc_compute;
  panel  a C5-shaped panel through brc_run_device: 1 000 sites at 50 000x from the counter-based generator, one complex record
         (REF 3 bp) per site whose ALTs are up to two allele strings of the host generator's identical copy of that site's
         reads (the first 512 of them), and one no read carries.

    python tools/vcf_complex_bench.py [--contig-len 2000000] [--step 20] [--panel-sites 1000] [--runs 3]
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

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    pl = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], text=True).strip()
    return name, pl


def records_of(reads, ref: str, positions, rng, ref_len):
    """(pos0, alleles) per position: the REF, up to two allele strings of spanning reads that differ from it, one made up."""
    import bisect
    import complex_rule
    out = []
    for p in positions:
        n = ref_len(rng)
        r = ref[p:p + n]
        alts = []
        for row in reads.rows[bisect.bisect_left(reads.starts, p - 160):bisect.bisect_left(reads.starts, p)][:64]:
            if row[1] <= p + n:
                continue
            f = complex_rule.resolve(row[4], row[0], p - 1, p + n)
            s = None if f is None else row[5][f[0] + 1:f[1]]
            if s and s != r and s not in alts and complex_rule._acgtn(s):
                alts.append(s)
            if len(alts) == 2:
                break
        out.append((p, [r] + alts + ["".join("ACGT"["ACGT".index(b) ^ 2] for b in r) + "A"]))
    return out


def wgs(args, res):
    import complex_rule
    from bam_readcount_b200 import synth
    from bam_readcount_b200.engine import Engine, pin_batch
    L = args.contig_len
    ref_a = synth.synth_reference(L, 1234)
    b = synth.synth_reads(ref_a, 30, seed=1234)
    ref = ref_a.tobytes().decode()
    rng = np.random.default_rng(1)
    recs = records_of(complex_rule.Reads(b), ref, range(1000, L - 1000, args.step), rng, lambda g: int(g.integers(1, 21)))
    pb = pin_batch(b)
    e = Engine(min_mapq=20, min_bq=20)
    e.set_reference(0, "chr1", L, ref.encode())
    ks, walls = [], []
    for _ in range(args.runs + 1):
        e.reset()
        e.begin_region(0, 999, L - 999, False)
        e.push_reads(pb)
        e.end_region()
        e.set_complex_queries([(0, p, len(al[0]), al) for p, al in recs])
        t0 = time.perf_counter()
        e.compute()
        walls.append(time.perf_counter() - t0)
        ks.append(e.stage_ms(5))
    d, c = e.complex_answers()
    res.update(wgs_reads=int(b.n_reads), wgs_records=len(recs), wgs_records_with_reads=int((d > 0).sum()),
               wgs_allele_counts_nonzero=int((c["count"] > 0).sum()), wgs_alleles=int(len(c)),
               wgs_stage5_ms=statistics.median(ks[1:]), wgs_compute_wall_s=statistics.median(walls[1:]))
    e.close()
    return b, ref_a, recs


def cli(args, res, b, ref_a, recs):
    """--vcf --vcf-complex against --vcf over the same VCF (samtools indexes the BAM; without it, not measured)."""
    from bam_readcount_b200 import build, synth
    from oracle.oracle import REF_SAMTOOLS
    if not os.path.exists(REF_SAMTOOLS):
        res.update(cli="not measured (no samtools to index the BAM)")
        return
    exe = build.build_cli()
    L = args.contig_len
    with tempfile.TemporaryDirectory() as d:
        synth.write_fasta(d + "/ref.fa", "chr1", ref_a)
        synth.write_sam(d + "/s.sam", b, [("chr1", L)])
        subprocess.check_call([REF_SAMTOOLS, "view", "-b", "-o", d + "/s.bam", d + "/s.sam"])
        subprocess.check_call([REF_SAMTOOLS, "index", d + "/s.bam"])
        with open(d + "/in.vcf", "w") as fh:
            fh.write("##fileformat=VCFv4.2\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tS1\n")
            for p, al in recs:
                fh.write(f"chr1\t{p + 1}\t.\t{al[0]}\t{','.join(al[1:])}\t.\t.\t.\tGT\t0/1\n")
        base = [exe, "-w", "0", "-q", "20", "-b", "20", "-f", d + "/ref.fa", "--vcf", d + "/in.vcf"]
        env = dict(os.environ, BRC_CLI_TIMING="1")
        wc, wp, kms = [], [], []
        for _ in range(args.runs):
            t0 = time.perf_counter()
            p = subprocess.run(base + ["--vcf-complex", d + "/s.bam"], capture_output=True, env=env, check=True)
            wc.append(time.perf_counter() - t0)
            kms.append(float([ln for ln in p.stderr.decode().splitlines() if "complex kernel" in ln][-1].split()[-2]))
            t0 = time.perf_counter()
            subprocess.run(base + [d + "/s.bam"], capture_output=True, env=env, check=True)
            wp.append(time.perf_counter() - t0)
        res.update(cli_vcf_complex_wall_s=statistics.median(wc), cli_vcf_wall_s=statistics.median(wp), cli_complex_kernel_ms=statistics.median(kms))


def panel(args, res):
    import torch
    import complex_rule
    from bam_readcount_b200 import synth_cb
    from bam_readcount_b200.engine import CRegion, Engine
    spec = synth_cb.Spec(seed=1234, mode=synth_cb.DEEP, n_libs=8, depth=50_000, site_stride=1000, n_sites=args.panel_sites,
                         contig_len=synth_cb.BLOCK_BP)
    n = args.panel_sites
    L = spec.deep_contig_len()
    dev = torch.device("cuda", 0)
    dw = synth_cb.DeviceWindow(spec, n * spec.depth, dev)
    stream = torch.cuda.Stream()
    dw.fill(0, 0, n, stream.cuda_stream)
    ref = spec.ref_host(0, 0, L).decode()
    rng = np.random.default_rng(2)
    recs = []
    for k in range(n):          # each site's ALTs: allele strings of the host generator's copy of that site's reads
        hb, _ = spec.window_host(0, k, k + 1)
        rows = complex_rule.Reads(hb.select(np.arange(min(hb.n_reads, 512))))
        recs += records_of(rows, ref, [spec.site_pos(k)], rng, lambda g: 3)
    regs = [CRegion(0, spec.site_pos(k), spec.site_pos(k) + 1, 1, k * spec.depth, (k + 1) * spec.depth, 2 * k, spec.site_pos(k) - 1, 2)
            for k in range(n)]
    e = Engine(max_cnt=100_000_000)
    e.set_reference(0, "chr1", L, ref.encode())
    ks, ks0 = [], []
    torch.cuda.synchronize()
    for _ in range(args.runs + 1):
        e.plan_device(regs, n * spec.depth, 1 << 20)
        e.set_complex_queries([(k, p, 3, al) for k, (p, al) in enumerate(recs)])
        e.run_device(dw.c_batch(), dw.t["region"].data_ptr(), stream.cuda_stream)
        e.fetch_device_results(stream.cuda_stream)
        ks.append(e.stage_ms(5))
        ks0.append(e.stage_ms(2))
    d, c = e.complex_answers()
    res.update(panel_sites=n, panel_reads=n * spec.depth, panel_stage5_ms=statistics.median(ks[1:]), panel_pileup_step_ms=statistics.median(ks0[1:]),
               panel_median_dp=int(np.median(d)), panel_alleles=int(len(c)), panel_allele_counts_nonzero=int((c["count"] > 0).sum()))
    e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--contig-len", type=int, default=2_000_000)
    ap.add_argument("--step", type=int, default=20)
    ap.add_argument("--panel-sites", type=int, default=1000)
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    name, pl = card()
    res = dict(card=name, power_limit_w=pl, runs=args.runs)
    b, ref_a, recs = wgs(args, res)
    cli(args, res, b, ref_a, recs)
    panel(args, res)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
