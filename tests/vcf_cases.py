"""Inputs of the --vcf tests: VCF text over the reference's test.bam fixture, its sample-column variants, and a BGZF writer."""
from __future__ import annotations

import os

import numpy as np

import bam_craft

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

HEAD = "##fileformat=VCFv4.2\n##contig=<ID=21>\n##FORMAT=<ID=GT,Number=1,Type=String,Description=\"Genotype\">\n"


def testbam_ref():
    """(window start, window bytes, contig length) of contig 21 as test_bam.npz stores it."""
    z = np.load(os.path.join(GOLDEN, "test_bam.npz"))
    return int(z["ref_win_beg"]), z["ref_win"].tobytes().decode("latin-1"), int(z["chrom_len"])


def fixture_records():
    """Records around the fixture's two covered sites: SNVs (all four bases, multi-allelic), insertions, deletions of several
    lengths, MNPs, '*', '<DEL>', lower case, a REF with an IUPAC letter, an N reference, a contig the BAM lacks and
    uncovered positions.  Each is (CHROM, POS, REF, ALT)."""
    wb, win, _ = testbam_ref()
    ref = lambda p, n=1: win[p - 1 - wb:p - 1 - wb + n].upper()        # 1-based
    out = []
    for site in (10402985, 10405200):
        for p in range(site - 6, site + 7):
            r = ref(p)
            alts = [b for b in "ACGT" if b != r]
            out.append(("21", p, r, ",".join(alts)))
            out.append(("21", p, r, r + "A," + r + "CT"))
            out.append(("21", p, ref(p, 2), r))
            out.append(("21", p, ref(p, 3), r + "," + ref(p + 1, 2)[::-1]))
        out.append(("21", site, ref(site).lower(), "a,<DEL>,*," + ref(site).lower() + "g"))
        out.append(("21", site + 1, ref(site + 1, 2), "TT,.,A"))
        out.append(("21", site, "N", "A,C"))
        out.append(("21", site, "R", "A"))
    out += [("chrZ", 100, "A", "C"), ("21", 10300000, "A", "G,AT"), ("21", 10300000, "AC", "A"), ("21", 1, "A", "G")]
    return out


def vcf_text(records, samples=("S1",), sites_only=False, pad=False) -> str:
    """A VCF of the records.  Sample columns hold a GT (the chosen sample's '.' when pad, so its values are padded)."""
    out = HEAD
    cols = "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO"
    out += cols + ("" if sites_only else "\tFORMAT\t" + "\t".join(samples)) + "\n"
    for k, (c, p, r, a) in enumerate(records):
        line = f"{c}\t{p}\trec{k}\t{r}\t{a}\t50\tPASS\tDP=10"
        if not sites_only:
            line += "\tGT:GQ\t" + "\t".join("." if pad and i == 0 else f"0/1:{k % 50}" for i in range(len(samples)))
        out += line + "\n"
    return out


def write_bgzf(path: str, data: bytes):
    """bgzip's format: BGZF members of at most 64 KiB and the empty end-of-file member."""
    with open(path, "wb") as fh:
        for i in range(0, len(data), 0xff00):
            fh.write(bam_craft.bgzf_member(data[i:i + 0xff00]))
        fh.write(bam_craft.bgzf_member(b""))


def write_fasta21(path: str):
    """ref.fa of contig 21: N everywhere except the window the fixture's reads touch."""
    from bam_readcount_b200 import synth
    wb, win, L = testbam_ref()
    seq = np.full(L, ord("N"), dtype=np.uint8)
    seq[wb:wb + len(win)] = np.frombuffer(win.encode("latin-1"), dtype=np.uint8)
    synth.write_fasta(path, "21", seq)
    return path
