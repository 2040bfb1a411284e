"""The alternative-allele site filter's rule, defined on the text: the test oracle of brc_set_site_filter and of brc-readcount's
--min-alt-count / --min-alt-fraction.

``select_lines`` parses bam-readcount's line grammar (with -p library blocks) and keeps a line iff one of its entries is an
alternative allele with count >= min_alt_count and count >= min_alt_fraction * depth.  A filtered run must print exactly
select_lines of the unfiltered output."""
import re

_ENTRY = re.compile(r"^([=ACGTN]|[+-][^:]*):(\d+):")
_NT16 = {"A": 1, "C": 2, "G": 4, "T": 8}

# (min_alt_count, min_alt_fraction) of the filtered runs: permissive, both bounds, fraction only, nothing passes
THRESHOLDS = [(1, 0.0), (2, 0.05), (1, 0.2), (10 ** 6, 0.0)]


def line_entries(fields):
    """(allele, count) of every allele entry of a line's fields after the depth column (library names and braces skipped)."""
    for f in fields:
        m = _ENTRY.match(f)
        if m:
            yield m.group(1), int(m.group(2))


def is_alt(allele: str, ref_base: str) -> bool:
    if allele[0] in "+-":
        return True
    if allele not in _NT16:
        return False                          # "=" and "N"
    return _NT16[allele] != _NT16.get(ref_base.upper(), 15)


def line_passes(line: str, min_alt_count: int, min_alt_fraction: float, ref_lookup=None) -> bool:
    f = line.split("\t")
    ref = ref_lookup(f[0], int(f[1])) if ref_lookup else f[2]
    depth = int(f[3])
    return any(is_alt(a, ref) and c >= min_alt_count and float(c) >= min_alt_fraction * float(depth) for a, c in line_entries(f[4:]))


def select_lines(text: str, min_alt_count: int, min_alt_fraction: float = 0.0, ref_lookup=None) -> str:
    """The lines of bam-readcount output `text` a site filter keeps.  ref_lookup(chrom, pos1) -> reference character; by
    default the line's own reference column."""
    return "".join(ln + "\n" for ln in text.splitlines() if line_passes(ln, min_alt_count, min_alt_fraction, ref_lookup))
