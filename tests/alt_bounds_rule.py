"""The site filter's entry bounds, defined on the text: the test oracle of brc_set_site_filter_bounds and of brc-readcount's
--alt-min / --alt-max.

A filtered line is printed iff one of its entries (any -p library block) is an alternative allele (site_filter_rule.is_alt) with
count >= min_alt_count and count >= min_alt_fraction * depth, and every bound that is set holds on that entry's printed fields.
A field's value is the decimal the line prints, in integer hundredths; bounds are {field name: (lo, hi)} in hundredths with
either side None."""
import re

from site_filter_rule import is_alt

FIELDS = ("count", "avg_mapping_quality", "avg_basequality", "avg_se_mapping_quality", "num_plus_strand", "num_minus_strand",
          "avg_pos_as_fraction", "avg_num_mismatches_as_fraction", "avg_sum_mismatch_qualities", "num_q2_containing_reads",
          "avg_distance_to_q2_start_in_q2_reads", "avg_clipped_length", "avg_distance_to_effective_3p_end")
_ENTRY = re.compile(r"^([=ACGTN]|[+-][^:]*)((?::-?\d+(?:\.\d\d)?){13})$")


def printed_hundredths(s: str) -> int:
    """'12' -> 1200, '0.12' -> 12, '-0.50' -> -50: the printed decimal in integer hundredths."""
    neg = s.startswith("-")
    whole, _, frac = s.lstrip("-").partition(".")
    v = int(whole) * 100 + int((frac + "00")[:2])
    return -v if neg else v


def entries(fields):
    """(allele, 13 values in hundredths) of every allele entry of a line's fields after the depth column."""
    for f in fields:
        m = _ENTRY.match(f)
        if m:
            yield m.group(1), [printed_hundredths(x) for x in m.group(2)[1:].split(":")]


def within(values, bounds) -> bool:
    for name, (lo, hi) in bounds.items():
        x = values[FIELDS.index(name)]
        if (lo is not None and x < lo) or (hi is not None and x > hi):
            return False
    return True


def line_passes_bounds(line: str, min_alt_count: int, min_alt_fraction: float, bounds: dict) -> bool:
    f = line.split("\t")
    depth = int(f[3])
    return any(is_alt(a, f[2]) and v[0] >= 100 * min_alt_count and float(v[0] // 100) >= min_alt_fraction * float(depth)
               and within(v, bounds) for a, v in entries(f[4:]))


def select_lines_bounds(text: str, min_alt_count: int, min_alt_fraction: float, bounds: dict) -> str:
    return "".join(ln + "\n" for ln in text.splitlines() if line_passes_bounds(ln, min_alt_count, min_alt_fraction, bounds))


def alt_values(text: str, min_alt_count: int = 1):
    """Per field, the sorted set of values that alternative entries of count >= min_alt_count print in `text`."""
    seen = [set() for _ in FIELDS]
    for ln in text.splitlines():
        f = ln.split("\t")
        for a, v in entries(f[4:]):
            if is_alt(a, f[2]) and v[0] >= 100 * min_alt_count:
                for k, x in enumerate(v):
                    seen[k].add(x)
    return [sorted(s) for s in seen]


# fpfilter-like sets: both strands seen, base quality, position in the read, mismatch burden, read-end distance
FPFILTER_SETS = [
    {"num_plus_strand": (100, None), "num_minus_strand": (100, None), "avg_basequality": (2000, None),
     "avg_pos_as_fraction": (10, None)},
    {"avg_mapping_quality": (2000, None), "avg_num_mismatches_as_fraction": (None, 5),
     "avg_sum_mismatch_qualities": (None, 5000), "avg_distance_to_effective_3p_end": (20, None)},
    {"count": (200, None), "avg_clipped_length": (1000, None), "num_q2_containing_reads": (None, 500),
     "avg_se_mapping_quality": (1000, 6000)},
]


def one_sided_sets(text: str, min_alt_count: int = 1):
    """For every field, one min bound and one max bound, each a value some alternative entry of `text` prints exactly (the
    median of the printed values), so inclusive and exclusive comparisons differ on the data.  Fields no entry prints: none."""
    out = []
    for name, vals in zip(FIELDS, alt_values(text, min_alt_count)):
        if vals:
            x = vals[len(vals) // 2]
            out += [{name: (x, None)}, {name: (None, x)}]
    return out
