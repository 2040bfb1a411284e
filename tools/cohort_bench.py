"""Wall time per sample of a cohort: K runs of `brc-readcount` (one process per sample) against one `--bam-list` run over the
same K samples.  Prints one JSON line per point, with the card name and power limit read in the same call.

Each sample is a seeded synthetic BAM (synth.synth_reads, a distinct seed per sample) on two contigs of 12 kb, written as SAM
and converted and indexed with oracle/_ref/samtools.  Library counts (0..4) and the @SQ order vary from sample to sample.  One
site list of about 2000 lines (single sites and short spans on both contigs) is used for every sample.  The two arms alternate,
--reps times each; every sample's output of the cohort run must equal its single run, byte for byte.

    python tools/cohort_bench.py [--points 64x30,64x500] [--reps 3] [--flags "-p"]
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

CONTIGS = (("ctgA", 12000, 101), ("ctgB", 12000, 102))        # name, length, reference seed


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
        return name, power
    except Exception as exc:                                   # no nvidia-smi: say so in the result rather than guess
        return f"unknown ({exc.__class__.__name__})", "unknown"


def _write_fasta(path, contigs):
    with open(path, "wb") as fa, open(path + ".fai", "w") as fai:
        off = 0
        for name, seq in contigs:
            head = f">{name}\n".encode()
            body = b"".join(seq[i:i + 60] + b"\n" for i in range(0, len(seq), 60))
            fa.write(head + body)
            fai.write(f"{name}\t{len(seq)}\t{off + len(head)}\t60\t61\n")
            off += len(head) + len(body)


def _make_sample(job):
    """One sample: seed k, n_libs = k % 5 (0: no @RG), contigs in header order swapped for odd k."""
    k, depth, d, samtools = job
    from bam_readcount_b200 import synth
    from bam_readcount_b200.batch import ReadBatch
    order = list(CONTIGS) if k % 2 == 0 else list(CONTIGS)[::-1]
    n_libs = k % 5
    parts = []
    for tid, (name, L, rs) in enumerate(order):
        ref = synth.synth_reference(L, rs)
        parts.append(synth.synth_reads(ref, depth, seed=1000 + 17 * k + tid, n_libs=max(n_libs, 1), tid=tid))
    sam, bam = os.path.join(d, f"s{k}.sam"), os.path.join(d, f"s{k}.bam")
    synth.write_sam(sam, ReadBatch.concat(parts), [(n, L) for n, L, _ in order], n_libs=max(n_libs, 1), read_group=n_libs > 0)
    subprocess.check_call([samtools, "view", "-b", "-o", bam, sam])
    subprocess.check_call([samtools, "index", bam])
    os.remove(sam)
    return bam


def make_point(d, K, depth, samtools, procs):
    import numpy as np
    from bam_readcount_b200 import synth
    fa = os.path.join(d, "ref.fa")
    _write_fasta(fa, [(n, synth.synth_reference(L, rs).tobytes()) for n, L, rs in CONTIGS])
    rng = np.random.default_rng(7)
    lines = []
    for name, L, _ in CONTIGS:
        for p in np.sort(rng.choice(np.arange(300, L - 300), 1000, replace=False)):
            lines.append(f"{name}\t{p}\t{p + (int(rng.integers(1, 20)) if rng.random() < 0.1 else 0)}\n")
    sites = os.path.join(d, "sites")
    open(sites, "w").write("".join(lines))
    with multiprocessing.Pool(procs) as pool:
        bams = pool.map(_make_sample, [(k, depth, d, samtools) for k in range(K)])
    return fa, sites, bams


def run_point(exe, d, K, depth, reps, flags, samtools, procs):
    fa, sites, bams = make_point(d, K, depth, samtools, procs)
    print(f"[cohort_bench] K={K} {depth}x: {K} samples written", file=sys.stderr, flush=True)
    args = [exe] + flags + ["-f", fa, "-l", sites]
    lst = os.path.join(d, "cohort.list")
    with open(lst, "w") as fh:
        for k, b in enumerate(bams):
            fh.write(f"{b}\t{d}/c{k}.out\t{d}/c{k}.err\n")
    single_t, cohort_t = [], []
    for rep in range(reps):
        t0 = time.perf_counter()
        for k, b in enumerate(bams):
            with open(f"{d}/s{k}.out", "wb") as o, open(f"{d}/s{k}.err", "wb") as e:
                subprocess.run(args + [b], stdout=o, stderr=e, check=True)
        single_t.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        subprocess.run(args + ["--bam-list", lst], check=True)
        cohort_t.append(time.perf_counter() - t0)
        print(f"[cohort_bench] K={K} {depth}x rep {rep}: single runs {single_t[-1]:.3f} s, cohort {cohort_t[-1]:.3f} s", file=sys.stderr, flush=True)
    equal = all(open(f"{d}/s{k}.out", "rb").read() == open(f"{d}/c{k}.out", "rb").read() and
                open(f"{d}/s{k}.err", "rb").read() == open(f"{d}/c{k}.err", "rb").read() for k in range(K))
    lines_out = sum(open(f"{d}/c{k}.out", "rb").read().count(b"\n") for k in range(K))
    # one run of each arm with BRC_CLI_TIMING: start-up vs region loop of the first and of a later sample
    env = dict(os.environ, BRC_CLI_TIMING="1")
    one = subprocess.run(args + [bams[0]], capture_output=True, env=env, check=True).stderr.decode()
    subprocess.run(args + ["--bam-list", lst], capture_output=True, env=env, check=True)
    timing = {"single_run": [ln for ln in one.splitlines() if ln.startswith("[brc timing] startup") or "region loop" in ln],
              "cohort_sample_0": [ln for ln in open(f"{d}/c0.err").read().splitlines() if ln.startswith("[brc timing] startup") or "region loop" in ln],
              "cohort_sample_1": [ln for ln in open(f"{d}/c1.err").read().splitlines() if ln.startswith("[brc timing] startup") or "region loop" in ln]}
    return dict(samples=K, depth=depth, site_list_lines=sum(1 for _ in open(sites)), printed_lines=lines_out, reps=reps, flags=" ".join(flags),
                single_s_per_sample=statistics.median(single_t) / K, cohort_s_per_sample=statistics.median(cohort_t) / K,
                single_total_s=[round(t, 3) for t in single_t], cohort_total_s=[round(t, 3) for t in cohort_t],
                outputs_equal=equal, timing=timing)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--points", default="64x30,64x500", help="comma-separated KxDEPTH points")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--flags", default="", help="extra brc-readcount options for every run")
    ap.add_argument("--procs", type=int, default=min(16, os.cpu_count() or 1), help="processes writing the sample BAMs")
    a = ap.parse_args()
    from bam_readcount_b200 import build
    from oracle.oracle import REF_SAMTOOLS
    if not os.path.exists(REF_SAMTOOLS):
        sys.exit("oracle/_ref/samtools is needed to write the sample BAMs (python __graft_entry__.py builds it)")
    build.build()
    exe = build.build_cli()
    name, power = card()
    for pt in a.points.split(","):
        K, depth = (int(x) for x in pt.lower().split("x"))
        with tempfile.TemporaryDirectory(prefix="brc_cohort_") as d:
            r = run_point(exe, d, K, depth, a.reps, a.flags.split(), REF_SAMTOOLS, a.procs)
        r.update(card=name, power_limit=power)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
