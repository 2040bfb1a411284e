"""Cases at the kernels' 32-bit edges (tests/test_edge32.py): CIGAR op indices past 2^31 and 2^32, and reads that run past
position 2^31 - 1.

cigar_offsets()      three regions whose non-simple reads reach every consumer of a read's CIGAR ops: K1 chunks that stage their
                     ops in shared memory and chunks with more than STAGE_CIGAR ops (global loads), a tile under >= 2048 reads
                     (deep_site_kernel), and a site-list line for the deep-site kernel forced with BRC_DEEP_MIN_READS=1.  The
                     device tests place the CIGAR pool 2^k - δ ops into a larger allocation; `cigar_target_delta` names the δ of
                     each target.
contig_end_2_31(k)   a contig of length 2^31 - 1 - k whose last sites are covered by reads overhanging its end (bam_endpos past
                     INT32_MAX).  The engine and the oracle get the last 100 kb of the contig as a reference window.

Every case is a dict in the tests/cases.py shape.  Deterministic: every builder takes its own seed."""
from __future__ import annotations

import functools

import numpy as np

from boundary_cases import K1_TILE, _case, _ref, _Reads

INT32_MAX = 2 ** 31 - 1

# 6 to 12 ops of every kind resolve_cigar2 walks (I, D, N, P, =, X, S); query length 148-150
MULTI_OP = ("30M2I20M3D25M1N20=3X50M", "5S40M1D30M2P2I30M4N41M", "25=1X24M2I30M2D20M1I47M", "10M1D10M1D10M1D10M1D10M1D100M",
            "50M1P1I49M3N49M1S", "3S20M2I20X1D30=2D40M3N33M")
_FEW_OP = ("150M", "150M", "150M", "60M1D90M", "150M", "150M", "30M2I118M", "150M")


def _site_reads(R, s, n, lib_mod=3):
    """n reads covering site s: the multi-op shapes from every start in s-140..s-1, and indel alleles anchored at s (an M op
    ending at s followed by I, D, or P then I), so resolve_cigar2's look-ahead at the next op runs at s."""
    for k in range(n):
        r = k % 10
        if r < 6:
            R.add(s - int(R.rng.integers(1, 141)), MULTI_OP[k % len(MULTI_OP)], lib=k % lib_mod, sub_rate=0.02)
        else:
            a = int(R.rng.integers(20, 120))                    # the M op covers [s - a + 1, s]
            tail, q_ins = (("2D", 0), ("3I", 3), ("1P2I", 2), ("1D", 0))[r - 6]
            R.add(s - a + 1, f"{a}M{tail}{150 - a - q_ins}M", lib=k % lib_mod, sub_rate=0.02)


@functools.lru_cache(maxsize=None)
def cigar_offsets(seed: int = 601):
    """Region 0 (argv, 2..20000): 150 bp reads every 10 bp; to 10 kb one read in four is non-simple (a 96-read K1 chunk holds
    <= STAGE_CIGAR ops: staged), from 12 kb every read is a 6-12 op MULTI_OP shape (chunks of ~800 ops: unstaged).
    Region 1 (site-list line 30001): 2100 reads over one site, deep_site_kernel by read count.
    Region 2 (site-list line 35001): 200 reads over one site, the deep-site kernel only when forced."""
    L = 40000
    ref = _ref(seed, L)
    R = _Reads(ref, seed)
    for k, p in enumerate(range(100, 10000, 10)):
        R.add(p, _FEW_OP[k % len(_FEW_OP)], lib=k % 3, mapq=int(R.rng.choice([60, 60, 30])), sub_rate=0.02)
    for k, p in enumerate(range(12000, 20000, 10)):
        R.add(p, MULTI_OP[k % len(MULTI_OP)], lib=k % 3, mapq=int(R.rng.choice([60, 60, 30])), sub_rate=0.02)
    _site_reads(R, 30000, 2100)
    _site_reads(R, 35000, 200)
    c = _case("cigar_offsets", ref, R.build(), [(0, 2, 20000), (0, 30001, 30001), (0, 35001, 35001)], site_list=True,
              modes=(True,), n_libs=3)
    return c


# region index and site-list mode of each CIGAR-offset target; "lookahead" is the deep tile again, with δ on its first indel
# read anchored at the site
CIGAR_TARGETS = dict(staged=(0, False), unstaged=(0, False), deep=(1, True), deep_forced=(2, True), lookahead=(1, True))


def _nonsimple(batch):
    """Per read: not FM_SIMPLE (more than one reference op, or an I / P op)."""
    co = batch.cigar_off.astype(np.int64) - int(batch.cigar_off[0])
    refops = np.isin(batch.cigar & 0xF, (0, 2, 3, 7, 8))
    ins = np.isin(batch.cigar & 0xF, (1, 6))
    n_ref = np.add.reduceat(refops.astype(np.int64), co[:-1])
    n_ins = np.add.reduceat(ins.astype(np.int64), co[:-1])
    return (n_ref != 1) | (n_ins > 0)


def cigar_target_delta(sub, target, chunks, site=None):
    """δ (ops of the region's batch before the boundary) of one target:
      staged       the boundary inside the op window of a staged-CIGAR K1 chunk, between two of its non-simple reads
      unstaged     the first op of the first non-simple read of the first chunk that does not stage its ops
      deep / deep_forced   the first op of the middle read of the site's reads
      lookahead    the first op of the first read that resolves to an indel at `site`"""
    co = sub.cigar_off.astype(np.int64)
    ns = _nonsimple(sub)
    if target == "staged":
        for c in chunks:
            idx = [i for i in range(c["r0"], c["r1"]) if ns[i]]
            if c["cstaged"] and len(idx) >= 4 and c["r0"] > 200:
                return int(co[idx[len(idx) // 2]]) - 1
    if target == "unstaged":
        for c in chunks:
            idx = [i for i in range(c["r0"], c["r1"]) if ns[i]]
            if not c["cstaged"] and idx:
                return int(co[idx[0]])
    if target in ("deep", "deep_forced"):
        return int(co[sub.n_reads // 2])
    if target == "lookahead":
        for i in range(sub.n_reads):
            if indel_at(sub, i, site) != 0:
                return int(co[i])
    raise AssertionError(f"no δ for {target}")


def indel_at(batch, i, site):
    """resolve_cigar2's indel length at `site` for read i (0 when it ends no M op there or the next op is not an indel)."""
    co = batch.cigar_off.astype(np.int64)
    ops = [(int(c) >> 4, int(c) & 15) for c in batch.cigar[co[i]:co[i + 1]]]
    x = int(batch.pos[i])
    for k, (ln, op) in enumerate(ops):
        if op in (0, 2, 3, 7, 8):
            if site < x + ln:
                if op in (0, 7, 8) and x + ln - 1 == site and k + 1 < len(ops):
                    l2, op2 = ops[k + 1]
                    if op2 in (1, 2):
                        return l2 if op2 == 1 else -l2
                    if op2 == 6:
                        return sum(l3 for l3, o3 in ops[k + 2:] if o3 == 1)
                return 0
            x += ln
    return 0


@functools.lru_cache(maxsize=None)
def contig_end_2_31(k: int = 0, seed: int = 611):
    """A contig of length 2^31 - 1 - k; the engine and the oracle get its last 100 kb (win_beg > 0).  About 4000 reads cover the
    last 20 kb; reads overhanging the end through an M op on both strands (simple 150M reads, so K1 pairs hot reads whose second
    one overhangs, and multi-op shapes); a deletion anchored at the site before the last (1D, then an M op past the end) and, when
    k >= 2, one anchored at the last site (a trailing 2D: D or N crossing the end before an M op would overflow the reference
    binary's int reference_position).  The argv region (argv_region) ends at the contig end with n_slots = 256 m + 2, so its last
    tile holds the last two sites: a warp window that reaches past INT32_MAX in pileup_kernel, a deep-site tile when forced.
    site_lines() are the last three positions."""
    L = INT32_MAX - k
    W = 100_000
    wb = L - W
    win = _ref(seed, W)
    R = _Reads(_Window(win, wb, L), seed)
    first_pos = L - K1_TILE * 78 - 2
    for p in np.sort(R.rng.integers(first_pos - 140, L - 150, 3600)):
        R.add(int(p), _FEW_OP[int(R.rng.integers(0, len(_FEW_OP)))], lib=int(R.rng.integers(0, 3)), mapq=int(R.rng.choice([60, 60, 20])),
              sub_rate=0.02)
    for j, p in enumerate(range(L - 149, L)):                   # overhanging the end through an M op
        # 8 ops whose last deletion ends at p + 61: from p > L - 62 on the simple 150M (the end is crossed by an M op only)
        cig = "20M2I20M1D20M1P1I85M" if j % 4 == 0 and p <= L - 62 else "150M"
        R.add(p, cig, lib=j % 3, flag=16 if j % 2 else 0, sub_rate=0.02)
    for j in range(6):
        a = 40 + j
        R.add(L - 1 - a, f"{a}M1D20M", lib=j % 3, sub_rate=0.0)  # deletion anchored at L - 2, M op past the end
        if k >= 2:
            R.add(L - a, f"{a}M2D", lib=j % 3, sub_rate=0.0)     # anchored at the last site, trailing deletion
    c = dict(name=f"end2_31_k{k}", contigs=[("c", L, win.tobytes(), wb)], batch=R.build(),
             regions=[(0, first_pos + 2, L)], site_list=False, modes=(False,), lib_names=[f"lib{i}" for i in range(3)], targets=[])
    return c


def site_lines(case):
    """The contig_end case with the site-list lines of its last three positions (1-based L-2, L-1, L)."""
    L = case["contigs"][0][1]
    return dict(case, name=case["name"] + "_l", regions=[(0, L - 2, L - 2), (0, L - 1, L - 1), (0, L, L)], site_list=True, modes=(True,))


class _Window:
    """The contig as edge_cases._read_from_ref indexes it: absolute positions, only [wb, L) held."""

    def __init__(self, win, wb, L):
        self.win, self.wb, self.L = win, wb, L

    def __len__(self):
        return self.L

    def __getitem__(self, i):
        return self.win[i - self.wb]


END_KS = (0, 1, 3, 30)
END_FLAGS = ("default", "perlib", "ic")


def jobs():
    """(case, flag-set name, flags, site_list mode, key) for the reference-binary anchor of the 2^31 cases."""
    import cases
    out = []
    for k in END_KS:
        c = contig_end_2_31(k)
        for fname in END_FLAGS:
            out.append((c, fname, cases.FLAG_SETS[fname], False, f"{c['name']}_{fname}"))
            out.append((site_lines(c), fname, cases.FLAG_SETS[fname], True, f"{c['name']}_l_{fname}"))
    return out
