"""--vcf against the pipeline it replaces: `brc-readcount -l <derived site list>` followed by parsing its text and writing the
counts into the VCF (tests/vcf_rule.py).  Prints one JSON line with the card's name and power limit.

Inputs: the synthetic 30x BAM of tools/sitelist_bench.py and a VCF with records every 20 bp: an SNV (the most frequent other
base of the site's line), and an insertion and a deletion wherever the line has one, so most alleles are present.

    python tools/vcf_bench.py [--contig-len 2000000] [--step 20] [--runs 3]
"""
from __future__ import annotations

import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    pl = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], text=True).strip()
    return name, pl


def make_vcf(text: str, ref: bytes) -> str:
    out = ["##fileformat=VCFv4.2\n", "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tS1\n"]
    for ln in text.splitlines():
        f = ln.split("\t")
        p, r = int(f[1]), f[2].upper()
        counts = {e.split(":")[0]: int(e.split(":")[1]) for e in f[4:]}
        alt = max((b for b in "ACGT" if b != r), key=lambda b: counts.get(b, 0))
        out.append(f"{f[0]}\t{p}\t.\t{r}\t{alt}\t.\t.\t.\tGT\t0/1\n")
        ins = [e for e in counts if e[0] == "+"]
        if ins and r in "ACGTN":
            out.append(f"{f[0]}\t{p}\t.\t{r}\t{r}{ins[0][1:]}\t.\t.\t.\tGT\t0/1\n")
        dels = [e for e in counts if e[0] == "-"]
        if dels:
            a = chr(ref[p - 2]).upper()
            out.append(f"{f[0]}\t{p - 1}\t.\t{a}{dels[0][1:].upper()}\t{a}\t.\t.\t.\tGT\t0/1\n")
    return "".join(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--contig-len", type=int, default=2_000_000)
    ap.add_argument("--step", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    from bam_readcount_b200 import build, synth
    from oracle.oracle import REF_SAMTOOLS
    import vcf_rule
    name, pl = card()
    exe = build.build_cli()
    L = args.contig_len
    with tempfile.TemporaryDirectory() as d:
        ref = synth.synth_reference(L, 1234)
        b = synth.synth_reads(ref, 30, seed=1234)
        synth.write_fasta(d + "/ref.fa", "chr1", ref)
        synth.write_sam(d + "/s.sam", b, [("chr1", L)])
        subprocess.check_call([REF_SAMTOOLS, "view", "-b", "-o", d + "/s.bam", d + "/s.sam"])
        subprocess.check_call([REF_SAMTOOLS, "index", d + "/s.bam"])
        os.remove(d + "/s.sam")
        with open(d + "/grid", "w") as fh:
            fh.write("".join(f"chr1\t{p}\t{p}\n" for p in range(1000, L - 1000, args.step)))
        base = [exe, "-w", "0", "-f", d + "/ref.fa"]
        grid = subprocess.run(base + ["-l", d + "/grid", d + "/s.bam"], capture_output=True, check=True).stdout.decode()
        vcf = make_vcf(grid, ref.tobytes())
        open(d + "/in.vcf", "w").write(vcf)
        open(d + "/derived", "w").write(vcf_rule.derive(vcf))
        env = dict(os.environ, BRC_CLI_TIMING="1")
        res = dict(card=name, power_limit_w=pl, reads=int(b.n_reads), records=vcf.count("\n") - 2, sites=vcf_rule.derive(vcf).count("\n"))
        walls_v, walls_l, walls_a, phases, alle = [], [], [], "", []
        for _ in range(args.runs):
            t0 = time.perf_counter()
            pv = subprocess.run(base + ["--vcf", d + "/in.vcf", d + "/s.bam"], capture_output=True, env=env, check=True)
            walls_v.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            pl_ = subprocess.run(base + ["-l", d + "/derived", d + "/s.bam"], capture_output=True, env=env, check=True)
            t1 = time.perf_counter()
            ann = vcf_rule.annotate(vcf, pl_.stdout.decode())
            walls_l.append(time.perf_counter() - t0)
            walls_a.append(time.perf_counter() - t1)
            err = pv.stderr.decode()
            phases = [ln for ln in err.splitlines() if "reference " in ln and "compute" in ln][-1]
            alle.append(float(re.search(r"allele kernels ([0-9.]+) ms", err).group(1)))
            assert pv.stdout.decode() == ann, "--vcf differs from the rule over -l derived"
        res.update(vcf_wall_s=statistics.median(walls_v), l_plus_annotate_wall_s=statistics.median(walls_l),
                   annotate_s=statistics.median(walls_a), vcf_timing=phases.split("] ", 1)[1], allele_kernel_ms=statistics.median(alle),
                   vcf_bytes=len(pv.stdout), text_bytes=len(pl_.stdout))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
