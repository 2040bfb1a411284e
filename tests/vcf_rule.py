"""The --vcf contract restated on text (DESIGN.md §12): which VCF records are counted, the site list they derive, and the VCF
`brc-readcount --vcf` writes, computed from the text of `brc-readcount -l <derived site list>` (or of the reference binary).

``derive(vcf_text)`` is the site list; ``annotate(vcf_text, readcount_text, sample=None, contigs=None)`` the annotated VCF:
``contigs`` is the BAM header's contig names (a record on another contig gets '.'), ``sample`` the --vcf-sample name.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

NT = "=ACGTN"
FORMAT_KEYS = ":BRC_DP:BRC_AD:BRC_ADF:BRC_ADR:BRC_AF"
HEADER = (
    '##FORMAT=<ID=BRC_DP,Number=1,Type=Integer,Description="brc-readcount depth of the site\'s line">\n'
    '##FORMAT=<ID=BRC_AD,Number=R,Type=Integer,Description="brc-readcount count of the REF and each ALT allele">\n'
    '##FORMAT=<ID=BRC_ADF,Number=R,Type=Integer,Description="brc-readcount plus-strand count of the REF and each ALT allele">\n'
    '##FORMAT=<ID=BRC_ADR,Number=R,Type=Integer,Description="brc-readcount minus-strand count of the REF and each ALT allele">\n'
    '##FORMAT=<ID=BRC_AF,Number=A,Type=Float,Description="brc-readcount BRC_AD of each ALT allele over BRC_DP">\n'
)


def _acgtn(s: str) -> bool:
    return len(s) > 0 and all(c in "ACGTN" for c in s)


def alleles(ref: str, alts: Sequence[str]) -> Tuple[Optional[int], Optional[str], List[Optional[str]]]:
    """(L offset or None when not counted, the REF entry's allele, per ALT the entry's allele or None when not countable).
    Entries are named as the text prints them: a base letter, "+BASES", or "-" + length (deletions match by length)."""
    ref = ref.upper()
    out: List[Optional[str]] = []
    for a in (x.upper() for x in alts):
        e = None
        if _acgtn(ref) and len(ref) == 1 and len(a) == 1 and _acgtn(a):
            e = a
        elif _acgtn(ref) and len(ref) == 1 and len(a) >= 2 and a[0] == ref[0] and _acgtn(a[1:]):
            e = "+" + a[1:]
        elif _acgtn(ref) and len(ref) >= 2 and a == ref[0]:
            e = "-%d" % (len(ref) - 1)
        out.append(e)
    if not any(e is not None for e in out):
        return None, None, out
    return (0 if len(ref) == 1 else 1), (ref[0] if len(ref) == 1 else ref[1]), out


def _records(vcf_text: str):
    for line in vcf_text.split("\n"):
        if line and not line.startswith("#"):
            yield line.split("\t")


def derive(vcf_text: str) -> str:
    """The derived site list: 'CHROM<TAB>L<TAB>L' per counted record, in file order."""
    out = []
    for c in _records(vcf_text):
        off, _, _ = alleles(c[3], c[4].split(","))
        if off is not None:
            L = int(c[1]) + off
            out.append(f"{c[0]}\t{L}\t{L}\n")
    return "".join(out)


def parse_lines(text: str) -> Dict[Tuple[str, int], Tuple[int, Dict[str, Tuple[int, int, int]]]]:
    """(chrom, 1-based pos) -> (depth, entry -> (count, plus, minus)) of a readcount text; deletions keyed '-<length>'."""
    out = {}
    for line in text.splitlines():
        f = line.split("\t")
        ent = {}
        for x in f[4:]:
            name, rest = x.split(":", 1)
            v = rest.split(":")
            key = ("-%d" % (len(name) - 1)) if name.startswith("-") else name.upper()
            ent[key] = (int(v[0]), int(v[4]), int(v[5]))
        out[(f[0], int(f[1]))] = (int(f[3]), ent)
    return out


def _values(ref_e, alt_e, line) -> str:
    dp, ent = line if line else (0, {})
    zero = (0, 0, 0)
    vals = [ent.get(ref_e, zero)] + [None if a is None else ent.get(a, zero) for a in alt_e]
    cols = [":".join([str(dp)] + [",".join("." if v is None else str(v[k]) for v in vals) for k in range(3)])]
    af = ",".join("." if v is None or dp == 0 else "%.6g" % (v[0] / dp) for v in vals[1:])
    return cols[0] + ":" + af


def annotate(vcf_text: str, readcount_text: str, sample: Optional[str] = None, contigs: Optional[Sequence[str]] = None) -> str:
    lines = parse_lines(readcount_text)
    out = []
    body = vcf_text.split("\n")
    if body and body[-1] == "":
        body = body[:-1]
    col = None
    for line in body:
        if line.startswith("##"):
            out.append(line + "\n")
            continue
        c = line.split("\t")
        if line.startswith("#CHROM"):
            out.append(HEADER)
            if len(c) == 8:
                out.append(line + "\tFORMAT\t" + sample + "\n")
            else:
                col = c.index(sample) if sample is not None else 9
                out.append(line + "\n")
            continue
        off, ref_e, alt_e = alleles(c[3], c[4].split(","))
        if off is None or (contigs is not None and c[0] not in contigs):
            vals = ".:.:.:.:."
        else:
            vals = _values(ref_e, alt_e, lines.get((c[0], int(c[1]) + off)))
        if col is None:
            out.append(line + "\t" + FORMAT_KEYS[1:] + "\t" + vals + "\n")
            continue
        keys = c[8].count(":") + 1
        s = c[col] + ":." * max(0, keys - (c[col].count(":") + 1))
        c[8] += FORMAT_KEYS
        c[col] = s + ":" + vals
        out.append("\t".join(c) + "\n")
    return "".join(out)
