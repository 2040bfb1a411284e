#!/usr/bin/env python
"""Regenerates tests/golden/ from the reference (run in the build container only).

Inputs: the reference's own fixtures under /root/reference/test-data (copied, they are data) and
the UNMODIFIED reference binary oracle/_ref/bam-readcount (oracle/build_ref.sh).  Outputs:
  expected_*                       the reference's four golden files, verbatim
  test_bam.npz, test_bam_bad_rg.npz  test.bam decoded to the compact batch + the reference
                                   window of contig 21 that its reads touch (ref.fa is 10.5 MB)
  ref_<case>_<flags>.txt.gz        reference-binary STDOUT on the deterministic synthetic cases
                                   of tests/cases.py (deletions, insertions, -q/-b, -i, -p, -d)
  edge_*.txt.gz                    reference-binary STDOUT on the hand-built edge-case reads
  fresh_fuzz_sha256.json, boundary_sha256.json
                                   SHA-256 of the reference binary's STDOUT on the fuzz seeds of test_differential_fuzz.py and
                                   on the capacity-boundary cases of boundary_cases.py (--boundary-only: only the latter)
  decode_sha256.json               SHA-256 of the reference binary's STDOUT and STDERR on the crafted BAMs of bam_craft.py
                                   (--decode-only: only this)
"""
import gzip
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import cases  # noqa: E402
import edge_cases  # noqa: E402
from bam_readcount_b200 import synth  # noqa: E402
from bam_readcount_b200.bamio import Fasta, read_bam  # noqa: E402
from oracle.oracle import REF_BIN, REF_SAMTOOLS, run_reference_binary  # noqa: E402

TD = "/root/reference/test-data"


def decode_fixture(bam, out):
    hdr, b = read_bam(os.path.join(TD, bam))
    fa = Fasta(os.path.join(TD, "ref.fa"))
    wb, we = 10402000, 10406000
    win = np.frombuffer(fa.fetch("21", wb, we), dtype=np.uint8)
    assert b.pos.min() >= wb and b.ref_end().max() <= we
    np.savez_compressed(os.path.join(HERE, out), tid=b.tid, pos=b.pos, flag=b.flag, mapq=b.mapq, lib=b.lib, l_qseq=b.l_qseq,
                        nm=b.nm, sm=b.sm, cigar_off=b.cigar_off, cigar=b.cigar, seq_off=b.seq_off, seq=b.seq,
                        qual_off=b.qual_off, qual=b.qual, ref_win=win, ref_win_beg=np.int64(wb),
                        chrom_len=np.int64(fa.length("21")), lib_names=np.array("\t".join(hdr.lib_names)))


def write_case_files(case, d):
    name, L, seq, wb = case["contigs"][0]
    if wb:      # the engine and the oracle get a window of the contig; the reference binary reads all of it
        seq = case["full_ref"]
    synth.write_fasta(os.path.join(d, "ref.fa"), name, np.frombuffer(seq, dtype=np.uint8))
    synth.write_sam(os.path.join(d, "s.sam"), case["batch"], [(name, L)], n_libs=len(case["lib_names"]),
                    read_group=case.get("read_group", True))
    _missing_qual_as_star(os.path.join(d, "s.sam"))
    subprocess.check_call([REF_SAMTOOLS, "view", "-b", "-o", os.path.join(d, "s.bam"), os.path.join(d, "s.sam")])
    subprocess.check_call([REF_SAMTOOLS, "index", os.path.join(d, "s.bam")])


def _missing_qual_as_star(path):
    """Quality bytes of 0xFF (a read stored with QUAL '*') come out of write_sam as spaces: write them as '*'.  SAM has no way to
    write 0xFF for only some bases of a read, so a batch holding such a read is refused."""
    with open(path) as fh:
        lines = fh.read().split("\n")
    for i, ln in enumerate(lines):
        f = ln.split("\t")
        if len(f) > 10 and not ln.startswith("@") and " " in f[10]:
            if f[10].strip(" "):
                raise ValueError(f"{f[0]}: quality 0xFF on some bases only cannot be written as SAM")
            f[10] = "*"
            lines[i] = "\t".join(f)
    with open(path, "w") as fh:
        fh.write("\n".join(lines))


def reference_stdout(case, flags, d, site_list):
    name = case["contigs"][0][0]
    argv = ["-w", "0", "-f", os.path.join(d, "ref.fa")] + cases.flags_to_argv(flags)
    if site_list:
        with open(os.path.join(d, "sites"), "w") as fh:
            for (_, b1, e1) in case["regions"]:
                fh.write(f"{name}\t{b1}\t{e1}\n")
        argv += ["-l", os.path.join(d, "sites"), os.path.join(d, "s.bam")]
    else:
        argv += [os.path.join(d, "s.bam")] + [f"{name}:{b1}-{e1}" for (_, b1, e1) in case["regions"]]
    out, err, rc = run_reference_binary(argv)
    assert rc == 0, err[-2000:]
    return out


def fresh_fuzz_jobs():
    """The fuzz cases of tests/test_differential_fuzz.py, run as site lists."""
    from test_differential_fuzz import SEEDS, _case
    jobs = []
    for seed in SEEDS:
        fc = _case(seed)
        for fname, fl in fc["flag_sets"].items():
            jobs.append((fc, fname, fl, True, f"{seed}_{fname}"))
    return jobs


def boundary_jobs():
    """The capacity-boundary cases of tests/boundary_cases.py: every flag set, in each region mode the case runs in."""
    import boundary_cases
    return boundary_cases.jobs()


def write_sha_file(jobs, out):
    sums, dirs = {}, {}
    for case, fname, fl, sl, key in jobs:
        if case["name"] not in dirs:
            dirs[case["name"]] = tempfile.mkdtemp()
            write_case_files(case, dirs[case["name"]])
        sums[key] = hashlib.sha256(reference_stdout(case, fl, dirs[case["name"]], sl).encode("latin-1")).hexdigest()
    with open(os.path.join(HERE, out), "w") as fh:
        json.dump(sums, fh, indent=1, sort_keys=True)


def write_decode_sha():
    """SHA-256 of the reference binary's STDOUT and STDERR on every crafted BAM of bam_craft.py that it reads as stored, per
    flag set of the decode tests."""
    import bam_craft
    sums = {}
    d = tempfile.mkdtemp()
    for f in bam_craft.write_corpus(d, REF_SAMTOOLS):
        if not f["vs_reference"]:
            continue
        for fname, argv in bam_craft.FLAG_SETS.items():
            out, err, rc = run_reference_binary(["-w", "1"] + argv + ["-f", f["fasta"], f["bam"]] + f["regions"])
            assert rc == 0, err[-2000:]
            sums[f"{f['name']}_{fname}"] = dict(stdout=hashlib.sha256(out.encode("latin-1")).hexdigest(),
                                                stderr=hashlib.sha256(err.encode("latin-1")).hexdigest())
    with open(os.path.join(HERE, "decode_sha256.json"), "w") as fh:
        json.dump(sums, fh, indent=1, sort_keys=True)


def main():
    assert os.path.exists(REF_BIN), "run oracle/build_ref.sh first"
    if "--decode-only" in sys.argv:
        write_decode_sha()
        return
    if "--boundary-only" in sys.argv:
        write_sha_file(boundary_jobs(), "boundary_sha256.json")
        return
    for f in ("expected_all_lib", "expected_per_lib", "expected_insertion_centric_all_lib",
              "expected_insertion_centric_per_lib"):
        shutil.copy(os.path.join(TD, f), os.path.join(HERE, f))
    decode_fixture("test.bam", "test_bam.npz")
    decode_fixture("test_bad_rg.bam", "test_bam_bad_rg.npz")

    # config 2b: the CRAM fixture through the reference binary (the reference ships no expected file for it)
    for flags, name in ((["-p"], "ref_cram_twolib_perlib.txt"), ([], "ref_cram_twolib_alllib.txt")):
        out, err, rc = run_reference_binary(flags + ["-l", "twolib_site_list.txt", "-f", "rand1k.fa", "twolib.sorted.cram"], cwd=TD)
        assert rc == 0
        with gzip.open(os.path.join(HERE, name + ".gz"), "wb", compresslevel=9) as fh:
            fh.write(out.encode("latin-1"))
        print(name, len(out.splitlines()), "lines")

    jobs = []
    syn = cases.synthetic_case(L=12000, depth=30, seed=11, regions=((0, 1000, 4000),), site_list=False)
    for fname, fl in cases.FLAG_SETS.items():
        jobs.append((syn, fname, fl, False, f"ref_syn_{fname}.txt"))
    deep = cases.deep_case(n_sites=3, depth=5000, seed=5)
    jobs.append((deep, "perlib_deep", dict(per_lib=True, max_cnt=100000000), True, "ref_deep_perlib.txt"))
    jobs.append((deep, "alllib_deep", dict(max_cnt=100000000), True, "ref_deep_alllib.txt"))
    for ec in edge_cases.all_cases():
        for fname, fl in ec["flag_sets"].items():
            jobs.append((ec, fname, fl, ec["site_list"], f"edge_{ec['name']}_{fname}.txt"))
    done = {}
    for case, fname, fl, sl, outname in jobs:
        key = case["name"]
        if key not in done:
            d = tempfile.mkdtemp()
            write_case_files(case, d)
            done[key] = d
        txt = reference_stdout(case, fl, done[key], sl)
        with gzip.open(os.path.join(HERE, outname + ".gz"), "wb", compresslevel=9) as fh:
            fh.write(txt.encode("latin-1"))
        print(outname, len(txt.splitlines()), "lines")

    # the fuzz seeds and the boundary cases: only the SHA-256 of the reference's STDOUT is kept
    write_sha_file(fresh_fuzz_jobs(), "fresh_fuzz_sha256.json")
    write_sha_file(boundary_jobs(), "boundary_sha256.json")
    write_decode_sha()


if __name__ == "__main__":
    main()
