"""--vcf-samples against one --vcf run per sample: N runs of `brc-readcount --vcf V --vcf-sample S_k BAM_k` (one process per
sample) against one `brc-readcount --vcf V --vcf-samples LIST` run over the same N samples.  Prints one JSON line per case, with
the card name and power limit read in the same call.

Each sample is a seeded synthetic BAM (synth.synth_reads, a distinct seed per sample) on two contigs, written as SAM and converted
and indexed with oracle/_ref/samtools.  The VCF has one column per sample and a few thousand records taken from the first
sample's own pileup text, as tests/test_vcf.py::test_cli_vcf_synthetic_indels builds them: at every STEP-th position an SNV (the
most frequent other base), and an insertion and a deletion wherever the line has one, so most alleles are present.  The two arms
alternate, --reps times each; `outputs_equal` says the single runs' columns, folded into one VCF, equal the one run's output.

    python tools/vcf_samples_bench.py [--cases 2,16] [--depth 30] [--contig-len 60000] [--step 30] [--reps 3]
"""
from __future__ import annotations

import argparse
import json
import multiprocessing
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
    if q.returncode != 0 or not q.stdout.strip():
        sys.exit("nvidia-smi could not read the card: this benchmark measures on a GPU")
    name, power = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
    return name, power


def _contigs(L):
    return (("ctgA", L, 201), ("ctgB", L, 202))              # name, length, reference seed


def _make_sample(job):
    k, depth, L, d, samtools = job
    from bam_readcount_b200 import synth
    from bam_readcount_b200.batch import ReadBatch
    parts = []
    for tid, (_, n, rs) in enumerate(_contigs(L)):
        parts.append(synth.synth_reads(synth.synth_reference(n, rs), depth, seed=3000 + 17 * k + tid, tid=tid))
    sam, bam = os.path.join(d, f"s{k}.sam"), os.path.join(d, f"s{k}.bam")
    synth.write_sam(sam, ReadBatch.concat(parts), [(n, ln) for n, ln, _ in _contigs(L)])
    subprocess.check_call([samtools, "view", "-b", "-o", bam, sam])
    subprocess.check_call([samtools, "index", bam])
    os.remove(sam)
    return bam


def make_vcf(exe, fa, bam, refs, L, step, names):
    """Records from `bam`'s own pileup text at every step-th position of both contigs."""
    sites = "".join(f"{n}\t{p}\t{p}\n" for n, _, _ in _contigs(L) for p in range(300, L - 300, step))
    with tempfile.NamedTemporaryFile("w", suffix=".sites", delete=False) as fh:
        fh.write(sites)
    text = subprocess.run([exe, "-w", "0", "-f", fa, "-l", fh.name, bam], capture_output=True, check=True).stdout.decode()
    os.remove(fh.name)
    cols = "\t".join("0/1" for _ in names)
    out = ["##fileformat=VCFv4.2\n", "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\t" + "\t".join(names) + "\n"]
    for ln in text.splitlines():
        f = ln.split("\t")
        c, p, r = f[0], int(f[1]), f[2].upper()
        counts = {e.split(":")[0]: int(e.split(":")[1]) for e in f[4:]}
        alt = max((b for b in "ACGT" if b != r), key=lambda b: counts.get(b, 0))
        out.append(f"{c}\t{p}\t.\t{r}\t{alt}\t.\t.\t.\tGT\t{cols}\n")
        ins = [e for e in counts if e[0] == "+"]
        if ins:
            out.append(f"{c}\t{p}\t.\t{r}\t{r}{ins[0][1:]}\t.\t.\t.\tGT\t{cols}\n")
        dels = [e for e in counts if e[0] == "-"]
        if dels:
            a = refs[c][p - 2]
            out.append(f"{c}\t{p - 1}\t.\t{a}{dels[0][1:].upper()}\t{a}\t.\t.\t.\tGT\t{cols}\n")
    return "".join(out)


def fold(singles):
    """One VCF from the single runs: header and columns 0-8 of the first, column 9 + k from run k."""
    runs = [s.decode().splitlines() for s in singles]
    out = []
    for i, ln in enumerate(runs[0]):
        if ln.startswith("#"):
            out.append(ln)
            continue
        out.append("\t".join(ln.split("\t")[:9] + [r[i].split("\t")[9 + k] for k, r in enumerate(runs)]))
    return ("\n".join(out) + "\n").encode()


def run_case(exe, d, n, a, samtools):
    from bam_readcount_b200 import synth
    L = a.contig_len
    fa = os.path.join(d, "ref.fa")
    refs = {}
    with open(fa, "wb") as fh, open(fa + ".fai", "w") as fai:
        off = 0
        for name, ln, rs in _contigs(L):
            seq = synth.synth_reference(ln, rs).tobytes()
            refs[name] = seq.decode()
            head = f">{name}\n".encode()
            body = b"".join(seq[i:i + 60] + b"\n" for i in range(0, ln, 60))
            fh.write(head + body)
            fai.write(f"{name}\t{ln}\t{off + len(head)}\t60\t61\n")
            off += len(head) + len(body)
    with multiprocessing.Pool(min(n, a.procs)) as pool:
        bams = pool.map(_make_sample, [(k, a.depth, L, d, samtools) for k in range(n)])
    names = ["TUMOR", "NORMAL"] if n == 2 else [f"S{k}" for k in range(n)]
    vcf = os.path.join(d, "in.vcf")
    text = make_vcf(exe, fa, bams[0], refs, L, a.step, names)
    open(vcf, "w").write(text)
    lst = os.path.join(d, "samples.tsv")
    with open(lst, "w") as fh:
        fh.write("".join(f"{nm}\t{b}\t{d}/m{k}.err\n" for k, (nm, b) in enumerate(zip(names, bams))))
    base = [exe, "-f", fa, "--vcf", vcf]
    single_t, multi_t, singles, multi = [], [], [], b""
    for rep in range(a.reps):
        t0 = time.perf_counter()
        singles = [subprocess.run(base + ["--vcf-sample", nm, b], capture_output=True, check=True).stdout for nm, b in zip(names, bams)]
        single_t.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        multi = subprocess.run(base + ["--vcf-samples", lst], capture_output=True, check=True).stdout
        multi_t.append(time.perf_counter() - t0)
        print(f"[vcf_samples_bench] {n} samples rep {rep}: single runs {single_t[-1]:.3f} s, one run {multi_t[-1]:.3f} s", file=sys.stderr, flush=True)
    timed = subprocess.run(base + ["--vcf-samples", lst], capture_output=True, check=True, env=dict(os.environ, BRC_CLI_TIMING="1")).stderr.decode()
    return dict(samples=n, depth=a.depth, contig_len=L, records=sum(1 for ln in text.splitlines() if not ln.startswith("#")), reps=a.reps,
                single_runs_s=statistics.median(single_t), one_run_s=statistics.median(multi_t),
                single_runs_total_s=[round(t, 3) for t in single_t], one_run_total_s=[round(t, 3) for t in multi_t],
                speedup=statistics.median(single_t) / statistics.median(multi_t), vcf_bytes=len(multi),
                outputs_equal=fold(singles) == multi, summary=[ln for ln in timed.splitlines() if "vcf-samples:" in ln])


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--cases", default="2,16", help="comma-separated sample counts")
    ap.add_argument("--depth", type=int, default=30)
    ap.add_argument("--contig-len", type=int, default=60000)
    ap.add_argument("--step", type=int, default=30, help="one pileup position per STEP bases becomes records")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--procs", type=int, default=min(16, os.cpu_count() or 1), help="processes writing the sample BAMs")
    a = ap.parse_args()
    from bam_readcount_b200 import build
    from oracle.oracle import REF_SAMTOOLS
    if not os.path.exists(REF_SAMTOOLS):
        sys.exit("oracle/_ref/samtools is needed to write the sample BAMs (python __graft_entry__.py builds it)")
    build.build()
    exe = build.build_cli()
    name, power = card()
    for n in (int(x) for x in a.cases.split(",")):
        with tempfile.TemporaryDirectory(prefix="brc_vcf_samples_") as d:
            r = run_case(exe, d, n, a, REF_SAMTOOLS)
        r.update(card=name, power_limit=power)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
