"""Inputs of the --vcf-complex tests: a hand-built BAM around one MNP (every way a read can or cannot span it), and synthetic
contigs with thousands of complex records whose ALTs are cut from the reads' own bases."""
from __future__ import annotations

import bisect
import os

import numpy as np

import bam_craft
import cases
import complex_rule
from bam_readcount_b200 import bamio, synth

L = 300
P = 100                      # 0-based first span base of the crafted MNP (POS 101); flanks 99 and 102


def crafted_ref() -> str:
    rng = np.random.default_rng(41)
    return "".join("ACGT"[x] for x in rng.integers(0, 4, L))


def _other(b: str) -> str:
    return "ACGT"[("ACGT".index(b) + 2) % 4]


def crafted_alleles():
    """(REF, MNP ALT, ALT with two bases inserted before the span, ALT with one base inserted after it)."""
    ref = crafted_ref()
    r = ref[P:P + 2]
    return r, _other(r[0]) + _other(r[1]), "GG" + r, r + "C"


def _seq(ref, pos, cig, subs=None, ins=None):
    """The read bases of an alignment: reference bases (subs: refpos -> base), inserted bases (ins: refpos before -> bases),
    'A' for soft clips."""
    subs, ins = subs or {}, ins or {}
    out, rp = [], pos
    for op, n in cig:
        if op in "M=X":
            out += [subs.get(rp + k, ref[rp + k]) for k in range(n)]
            rp += n
        elif op == "I":
            out.append(ins[rp - 1])
        elif op == "S":
            out.append("A" * n)
        elif op in "DN":
            rp += n
    return "".join(out)


def crafted_reads():
    """(name, pos, CIGAR, seq, qual, flag, mapq, S): S the allele string of the read under the default flags (None: it does
    not span or is dropped by the flag filter)."""
    ref = crafted_ref()
    r, mnp, ins_l, ins_r = crafted_alleles()
    alt = {P: mnp[0], P + 1: mnp[1]}
    q = lambda n, low=None: [5 if k == low else 30 for k in range(n)]
    rows = []

    def add(name, pos, cig, subs=None, ins=None, low=None, flag=0, mapq=60, s=None):
        c = bam_craft.parse_cigar(cig)
        seq = _seq(ref, pos, c, subs, ins)
        rows.append((name, pos, cig, seq, q(len(seq), low), flag, mapq, s))
    add("mnp_M", 80, "40M", alt, s=mnp)
    add("mnp_eqx", 80, "20=2X18=", alt, s=mnp)
    add("mnp_1D1I", 80, "20M1D1I19M", {P + 1: mnp[1]}, {P: mnp[0]}, s=mnp)
    add("ins_left_flank", 80, "20M2I20M", ins={P - 1: "GG"}, s=ins_l)
    add("ins_right_flank", 80, "22M1I18M", ins={P + 1: "C"}, s=ins_r)
    add("right_flank_soft_clipped", 80, "22M18S", s=None)
    add("left_flank_deleted", 80, "19M1D20M", s=None)
    add("right_flank_skipped", 80, "22M3N18M", s=None)
    add("ends_on_right_flank", 80, "23M", s=r)
    add("ends_before_right_flank", 80, "22M", s=None)
    add("low_quality_inside", 80, "40M", low=20, s=r)
    add("low_quality_outside", 80, "40M", low=10, s=r)
    add("reverse", 80, "40M", alt, flag=16, s=mnp)
    add("other_haplotype", 80, "40M", {P: mnp[0]}, s=mnp[0] + r[1])
    add("iupac_base", 80, "40M", {P + 1: "R"}, s=r[0] + "N")
    add("duplicate", 80, "40M", alt, flag=1024, s=None)
    add("secondary", 80, "40M", alt, flag=256, s=None)
    add("qc_fail", 80, "40M", alt, flag=512, s=None)
    add("low_mapq", 81, "40M", alt, mapq=5, s=mnp)
    add("reverse_ref", 82, "40M", flag=16, s=r)
    add("left_flank_soft_clipped", 100, "5S35M", s=None)          # reads are in position order
    return rows


def crafted_records():
    """(CHROM, POS, REF, ALT) of the crafted VCF: the MNP with its three ALTs, the IUPAC read's allele (its R reads as N) and a
    '*', a mixed SNV / complex record, an
    SNV and a deletion counted per site, and a complex record past the contig's end."""
    ref = crafted_ref()
    r, mnp, ins_l, ins_r = crafted_alleles()
    return [("chr1", 90, ref[89], _other(ref[89])), ("chr1", P + 1, r, f"{mnp},{ins_l},{ins_r},{r[0]}N,*"),
            ("chr1", P + 1, r[0], f"{_other(r[0])},{_other(r[0])}{r[1]}"), ("chr1", P, ref[P - 1:P + 1], ref[P - 1]),
            ("chr1", P + 1, ref[P:P + 3], mnp), ("chr1", L - 1, ref[L - 2:], "TT")]


def write_crafted(d: str, samtools=None):
    """The crafted BAM (indexed when samtools is given) and FASTA in d: (bam path, fasta path)."""
    recs = [bam_craft.record(n, 0, p, bam_craft.parse_cigar(c), s, q, flag=f, mapq=m) for n, p, c, s, q, f, m, _ in crafted_reads()]
    bam = bam_craft.write_bam(os.path.join(d, "crafted.bam"), "@HD\tVN:1.6\tSO:coordinate\n", [("chr1", L)], recs, index=samtools)
    fa = os.path.join(d, "crafted.fa")
    synth.write_fasta(fa, "chr1", np.frombuffer(crafted_ref().encode(), dtype=np.uint8))
    return bam, fa


def crafted_case(d: str) -> dict:
    """The crafted BAM decoded by bamio.read_bam, as a tests/cases.py case with one site-list region per record."""
    bam, _ = write_crafted(d)
    hdr, batch = bamio.read_bam(bam)
    regions = [(0, p, p) for _, p, _, _ in crafted_records()]
    return dict(name="complex_crafted", contigs=[("chr1", L, crafted_ref().encode(), 0)], batch=batch, regions=regions,
                site_list=True, lib_names=[])


def synthetic_records(case, n_records: int, seed: int, every: int = 20):
    """Records on the case's first contig, one every `every` bp: complex ones with REF lengths 1-20 and ALTs cut from a
    spanning read's bases (so most have reads), and every fifth an SNV counted per site."""
    rng = np.random.default_rng(seed)
    name, clen, seq, wb = case["contigs"][0]
    ref = seq.decode()
    reads = complex_rule.Reads(case["batch"])
    out = []
    for k in range(n_records):
        pos0 = 300 + k * every
        if pos0 + 25 >= clen - 300:
            break
        if k % 5 == 4:
            out.append((name, pos0 + 1, ref[pos0], _other(ref[pos0])))
            continue
        n = int(rng.integers(1, 21))
        r = ref[pos0:pos0 + n]
        alts = []
        lo = bisect.bisect_left(reads.starts, pos0 - 160)
        for row in reads.rows[lo:lo + 40]:
            if row[0] > pos0 - 1 or row[1] <= pos0 + n:
                continue
            f = complex_rule.resolve(row[4], row[0], pos0 - 1, pos0 + n)
            if f is not None and f[1] - f[0] > 1:
                s = row[5][f[0] + 1:f[1]]
                if s != r and s not in alts and complex_rule._acgtn(s):
                    alts.append(s)
        alts = alts[:2] + ["".join(_other(b) for b in r) + "A"]       # and one no read carries
        out.append((name, pos0 + 1, r, ",".join(alts)))
    return out


def rule_answers(case, records, flags, reads=None):
    """complex_rule.count of every complex record of `records` over the reads of the record's line that the engine admits:
    {(pos0, ref_len, alleles): (DP, counts)}.  `reads`: one complex_rule.Reads for all records (every read admitted)."""
    from bam_readcount_b200.engine import admitted
    out = {}
    _, clen, _, _ = case["contigs"][0]
    for chrom, pos, ref, alt in records:
        cx = complex_rule.complex_alleles(pos, ref, alt.split(","))
        if cx is None:
            continue
        rr = reads
        if rr is None:
            tid, _, _, sub = cases.region_reads(case, 0, pos, pos)
            rr = complex_rule.Reads(sub, admitted(sub, tid, flags.get("max_cnt", 10_000_000)))
        al = [cx[0]] + [a for a in cx[1] if a is not None]
        out[(pos - 1, len(cx[0]), tuple(al))] = complex_rule.count(rr, pos - 1, len(cx[0]), al, flags.get("min_mapq", 0),
                                                                  flags.get("min_bq", 0), clen)
    return out
