"""The --vcf-complex rule restated on decoded reads (DESIGN.md §12 "MNP and complex records").

A record is complex when POS >= 2, REF (upper-cased) is A/C/G/T/N letters and one of its ALTs is an A/C/G/T/N string that the
per-site rule (tests/vcf_rule.py) cannot count.  Its span is the 0-based reference positions [P, P + n) (P = POS - 1, n =
len(REF)); its flanks are P - 1 and P + n.  A read spans it when both flanks are aligned to read bases by M, = or X; its allele
string S is the read bases strictly between the two flank query positions (inserted bases included; IUPAC codes read as N).
A read counts when it is admitted (engine.admitted), not dropped by -q or the flag filter, spans the record and has no base
of S below -b.  BRC_DP is the reads that count; BRC_AD per allele the counted reads whose S equals it, split by strand.

``resolve(cigar_words, pos, left, right)`` is the flank walk (the twin of brc_complex.cuh), ``count(reads, ...)`` the
answer of one record, ``derive`` / ``annotate`` the --vcf-complex site list and VCF.
"""
from __future__ import annotations

import bisect
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

import vcf_rule

CANON = "=ACNGNNNTNNNNNNN"          # nibble -> the letter bam_nt16_canonical_table gives it ("=ACGTN")
FLAG_FILTER = 4 | 256 | 512 | 1024


def _acgtn(s: str) -> bool:
    return len(s) > 0 and all(c in "ACGTN" for c in s)


def complex_alleles(pos: int, ref: str, alts: Sequence[str]) -> Optional[Tuple[str, List[Optional[str]]]]:
    """(REF, per ALT the allele or None when it is not A/C/G/T/N) of a complex record; None when the record is not complex."""
    ref = ref.upper()
    ups = [a.upper() for a in alts]
    _, _, per_site = vcf_rule.alleles(ref, ups)
    if pos < 2 or not _acgtn(ref) or not any(e is None and _acgtn(a) for e, a in zip(per_site, ups)):
        return None
    return ref, [a if _acgtn(a) else None for a in ups]


def resolve(cigar: Sequence[int], pos: int, left: int, right: int) -> Optional[Tuple[int, int]]:
    """Query positions of the two flanks, or None when the read does not span: a map from each match-aligned reference
    position to its query position."""
    at: Dict[int, int] = {}
    rp, qp = pos, 0
    for w in cigar:
        op, ln = int(w) & 0xF, int(w) >> 4
        if op in (0, 7, 8):
            for k in range(ln):
                at[rp + k] = qp + k
            rp += ln
            qp += ln
        elif op in (1, 4):
            qp += ln
        elif op in (2, 3):
            rp += ln
    if left in at and right in at:
        return at[left], at[right]
    return None


class Reads:
    """One region's admitted reads, decoded once: per read its start, end, strand, CIGAR, bases and qualities."""

    def __init__(self, batch, idx=None):
        idx = np.arange(batch.n_reads) if idx is None else np.asarray(idx)
        end = batch.ref_end()
        nib = np.empty(2 * batch.seq.shape[0], np.uint8)
        nib[0::2], nib[1::2] = batch.seq >> 4, batch.seq & 0xF
        letters = np.frombuffer(CANON.encode(), np.uint8)[nib].tobytes().decode()    # every base of the pool, as S spells it
        quals = batch.qual.tobytes()
        self.rows = []
        for i in idx.tolist():
            c0, c1 = int(batch.cigar_off[i]), int(batch.cigar_off[i + 1])
            s0, q0, lq = 2 * int(batch.seq_off[i]), int(batch.qual_off[i]), int(batch.l_qseq[i])
            self.rows.append((int(batch.pos[i]), int(end[i]), int(batch.flag[i]), int(batch.mapq[i]),
                              batch.cigar[c0:c1].tolist(), letters[s0:s0 + lq], quals[q0:q0 + lq]))
        self.rows.sort(key=lambda r: r[0])
        self.starts = [r[0] for r in self.rows]
        self.span = max([r[1] - r[0] for r in self.rows], default=0)


def count(reads: Reads, pos0: int, n: int, alleles: Sequence[str], min_mapq=0, min_bq=0, chrom_len=None):
    """(DP, [(count, plus, minus) per allele]) of the record whose span is [pos0, pos0 + n)."""
    left, right = pos0 - 1, pos0 + n
    dp, cnt = 0, [[0, 0] for _ in alleles]
    if chrom_len is not None and right >= chrom_len:
        return 0, [(0, 0, 0) for _ in alleles]
    for r in reads.rows[bisect.bisect_left(reads.starts, right - reads.span):bisect.bisect_right(reads.starts, left)]:
        p, e, flag, mapq, cig, seq, qual = r
        if e <= right or flag & FLAG_FILTER or mapq < min_mapq:
            continue
        f = resolve(cig, p, left, right)
        if f is None:
            continue
        s = seq[f[0] + 1:f[1]]
        if any(q < min_bq for q in qual[f[0] + 1:f[1]]):
            continue
        dp += 1
        for k, a in enumerate(alleles):
            if s == a:
                cnt[k][0] += 1
                cnt[k][1] += 0 if flag & 16 else 1
    return dp, [(c, p, c - p) for c, p in cnt]


def derive(vcf_text: str) -> str:
    """The --vcf --vcf-complex site list: vcf_rule.derive's line for a per-site record, 'CHROM POS POS' for a complex one."""
    out = []
    for c in vcf_rule._records(vcf_text):
        if complex_alleles(int(c[1]), c[3], c[4].split(",")) is not None:
            out.append(f"{c[0]}\t{c[1]}\t{c[1]}\n")
        else:
            off, _, _ = vcf_rule.alleles(c[3], c[4].split(","))
            if off is not None:
                L = int(c[1]) + off
                out.append(f"{c[0]}\t{L}\t{L}\n")
    return "".join(out)


def complex_values(dp: int, counts, alts) -> str:
    """The five FORMAT values of a complex record: counts holds the REF's and each A/C/G/T/N ALT's (count, plus, minus)."""
    it = iter(counts[1:])
    vals = [counts[0]] + [None if a is None else next(it) for a in alts]
    cols = [str(dp)] + [",".join("." if v is None else str(v[k]) for v in vals) for k in range(3)]
    af = ",".join("." if v is None or dp == 0 else "%.6g" % (v[0] / dp) for v in vals[1:])
    return ":".join(cols) + ":" + af


def annotate(vcf_text: str, readcount_text: str, answers, sample: Optional[str] = None,
             contigs: Optional[Sequence[str]] = None) -> str:
    """vcf_rule.annotate, with each complex record's five values from answers(chrom, pos0, ref_len, alleles) -> (DP, counts)
    (alleles: the REF, then each A/C/G/T/N ALT); a record on a contig the BAM lacks keeps '.'."""
    out = vcf_rule.annotate(vcf_text, readcount_text, sample=sample, contigs=contigs).split("\n")
    col = None
    data = (k for k, ln in enumerate(out) if ln and not ln.startswith("#"))
    for line in vcf_text.split("\n"):
        if line.startswith("#CHROM"):
            h = line.split("\t")
            col = 9 if len(h) == 8 or sample is None else h.index(sample)
        if not line or line.startswith("#"):
            continue
        k = next(data)
        c = line.split("\t")
        cx = complex_alleles(int(c[1]), c[3], c[4].split(","))
        if cx is None or (contigs is not None and c[0] not in contigs):
            continue
        ref, alts = cx
        dp, counts = answers(c[0], int(c[1]) - 1, len(ref), [ref] + [a for a in alts if a is not None])
        o = out[k].split("\t")
        head = o[col].rsplit(":", 5)
        o[col] = (head[0] + ":" if len(head) == 6 else "") + complex_values(dp, counts, alts)
        out[k] = "\t".join(o)
    return "\n".join(out)
