"""Seeded cases that straddle the kernels' hard capacities and fast-path predicates (DESIGN.md §4):
K0's shared-memory stage (128 reads, K0_QUAL_CAP / K0_SEQ_CAP, the packed reference window), K1's chunks (STAGE_READS
descriptors, STAGE_QUAL / STAGE_SEQ bytes, STAGE_CIGAR ops) and warp windows, the reciprocal-division fast path
(FASTDIV_MAX), the narrow packed record (8-bit depth, 16-bit sums), the deep-site kernel's 256-read blocks and insertion
cache, and byte values the usual workloads never carry (QUAL '*', MAPQ 255, negative SM).

Every case is a dict in the tests/cases.py shape plus
  targets   the limits it straddles (tests/test_kernel_boundaries.py recomputes the kernels' decisions and checks that each
            target is hit on both sides)
  modes     the region modes it runs in: True = site list (-l), False = argv regions
  full_ref  the whole contig when the case hands the engine only a window of it (win_beg > 0); the reference binary reads
            the whole FASTA
Deterministic: every builder takes its own seed."""
from __future__ import annotations

import functools
import re

import numpy as np

import edge_cases
from bam_readcount_b200.batch import BatchBuilder

K1_TILE = 256


def _ops(cigar: str):
    return [(int(n), o) for n, o in re.findall(r"(\d+)([MIDNSHP=XB])", cigar)]


def _quals(rng, n, reverse, q2_tail=True):
    q = rng.choice(np.array([40, 37, 33, 30, 25, 20], np.uint8), size=n)
    if q2_tail and rng.random() < 0.5:
        t = int(rng.integers(1, max(2, n // 8)))
        if reverse:
            q[:t] = 2
        else:
            q[n - t:] = 2
    return q


class _Reads:
    """Collects SAM-like records over one reference and builds the batch in file (position) order."""

    def __init__(self, ref, seed):
        self.ref = ref
        self.rng = np.random.default_rng(seed)
        self.recs = []

    def add(self, pos, cigar, *, flag=None, mapq=60, lib=0, qual=None, nm=1, sm=None, sub_rate=0.01, seq=None, q2_tail=True):
        rng = self.rng
        if flag is None:
            flag = 16 if rng.random() < 0.5 else 0
        ops = _ops(cigar)
        if seq is None:
            seq = edge_cases._read_from_ref(rng, self.ref, int(pos), ops, sub_rate)
        lq = len(seq)
        if qual is None:
            qual = _quals(rng, lq, bool(flag & 16), q2_tail)
        self.recs.append(dict(tid=0, pos=int(pos), flag=int(flag), mapq=int(mapq), lib=lib, cigar=cigar, seq=seq,
                              qual=np.asarray(qual, np.uint8), nm=nm, sm=sm, qname=f"b{len(self.recs)}"))

    def build(self):
        self.recs.sort(key=lambda r: r["pos"])      # stable: equal positions keep insertion order
        bb = BatchBuilder()
        for r in self.recs:
            bb.add_sam(**r)
        return bb.build()


def _ref(seed, L):
    return np.random.default_rng(seed).choice(np.frombuffer(b"ACGT", np.uint8), size=L)


def _case(name, ref, batch, regions, *, site_list=True, modes=(True,), n_libs=3, targets=(), win_beg=0):
    L = int(ref.shape[0])
    c = dict(name=name, contigs=[("c", L, ref[win_beg:].tobytes(), win_beg)], batch=batch, regions=list(regions),
             site_list=site_list, modes=tuple(modes), lib_names=[f"lib{i}" for i in range(n_libs)], targets=list(targets))
    if win_beg:
        c["full_ref"] = ref.tobytes()
    return c


def length_ladder(seed=401):
    """Uniform 128-read blocks of 152, 153, 160 and 161 bp (K1's chunk shrink starts at 153, K0's stage holds 160), then mixed
    blocks of 250-2049 bp around FASTDIV_MAX, with clipped lengths of 2048 / 2049."""
    L = 40000
    ref = _ref(seed, L)
    R = _Reads(ref, seed)
    base = 200
    for lq in (152, 153, 160, 161):
        for p in np.sort(R.rng.integers(base, base + 120, 128)):
            R.add(int(p), f"{lq}M", lib=int(R.rng.integers(0, 3)))
        base += 1200
    mixed = ["250M", "1000M", "2047M", "2048M", "2049M", "1S2047M", "1S2048M", "1S2049M", "2048M1S", "3S2045M", "2050M"]
    for k in range(2 * 128):
        cig = mixed[k % len(mixed)]
        R.add(base + 40 * k, cig, lib=int(R.rng.integers(0, 3)), sub_rate=0.005)
    return _case("ladder", ref, R.build(), [(0, 1, L)], targets=["k0_qual_cap", "k1_stage_shrink", "fastdiv_len", "fastdiv_clen"])


def clip_numerators(seed=402):
    """FM_HOT reads shaped nH mS kM (the soft clip after a hard clip counts as a right clip, so qpos - left_clip runs far past
    clipped_length), both strands, next to the controls mS kM nS and kM mS."""
    L = 8000
    ref = _ref(seed, L)
    R = _Reads(ref, seed)
    shapes = ["5H100S10M", "3H1000S40M", "2H2000S30M", "1H2038S10M", "7H500S60M2H", "100S10M5S", "40M1000S", "1000S40M", "10M2000S"]
    for k in range(600):
        cig = shapes[k % len(shapes)]
        p = 300 + (k // 3) * 30 + int(R.rng.integers(0, 20))
        R.add(p, cig, flag=16 if (k // len(shapes)) % 2 else 0, lib=int(R.rng.integers(0, 3)))
    return _case("numerators", ref, R.build(), [(0, 1, L)], targets=["fastdiv_numerator"])


def ref_window(win_beg, L, seed):
    """Reads to and past the contig end (L mod 4 varies), a contig window starting at win_beg, 1.5 kb reads in one K0 block
    (ops past the staged reference window) and a sparse block spanning more than 8192 bases (reference not staged)."""
    ref = _ref(seed, L)
    R = _Reads(ref, seed)
    p0 = win_beg + 20
    for k in range(128):        # block 0: dense, with 1.5 kb multi-op reads at its end
        if k >= 120:
            R.add(p0 + 300 + k, "500M2D500M1I499M", lib=k % 3, sub_rate=0.02)
        else:
            R.add(p0 + 2 * k, "100M", lib=k % 3, sub_rate=0.03)
    for k in range(128):        # block 1: sparse, first and last start > 8192 bases apart
        R.add(p0 + 2000 + 80 * k, "60M", lib=k % 3, sub_rate=0.03)
    end0 = win_beg + 13000
    for k in range(128):        # block 2: runs to and past the contig end
        p = end0 + 30 * k
        if p + 50 >= L:
            p = L - 60 + (k % 70)
        R.add(min(p, L - 1), "4S50M3S" if k % 5 else "50M", lib=k % 3, sub_rate=0.03)
    regions = [(0, win_beg + 2, L)]     # the pileup starts one position before the region: first_pos = win_beg
    return _case(f"refwin_{win_beg}_{L % 4}", ref, R.build(), regions, modes=(True, False), site_list=True,
                 targets=["k0_ref_window"], win_beg=win_beg)


def chunk_geometry(seed=404):
    """Tiles holding exactly 96, 97 and 192 reads; hot runs of odd and even length ending at a chunk boundary; reads starting at
    wfirst+31 / wfirst+32 and ending at wfirst / wfirst+1; reads starting at tile edges; more than 32 leading reads that end
    before the last warp's window; library-less reads inside hot runs; chunks just under and over STAGE_CIGAR ops."""
    L = 12 * 2 * K1_TILE + 600
    ref = _ref(seed, L)
    R = _Reads(ref, seed)
    tile = lambda t: 2 * t * K1_TILE      # every other tile holds reads, so each tile's read range is exactly its own reads

    def fill(t, n, nonhot=(), libless=(), cig="50M"):
        for k in range(n):
            p = tile(t) + 10 + (k * 190) // max(1, n)
            if k in nonhot:
                R.add(p, "25M1I24M", lib=k % 3)            # not FM_HOT: breaks a hot run
            else:
                R.add(p, cig, lib=None if k in libless else k % 3)
    fill(0, 96, nonhot={0})              # odd hot run (95) ends the chunk: A = the 96th read, B = the sentinel
    fill(1, 96)                          # even hot run ends the chunk
    fill(2, 97, nonhot={50})             # second chunk of one read
    fill(3, 192, nonhot={0, 95})         # two full chunks
    fill(4, 96, libless={31, 60})        # -p: a library-less read inside a hot run
    # warp-window edges: reads start at wfirst+31 / wfirst+32 and end at wfirst / wfirst+1 (wfirst = pos0 + 32 w)
    t5 = tile(5)
    for w in (1, 3, 6):
        wf = t5 + 32 * w
        for d in (31, 32, 31, 32):
            R.add(wf + d, "40M", lib=w % 3)
        for e in (0, 1, 0, 1):
            R.add(wf + e - 30, "30M", lib=(w + 1) % 3)
    # tile edges: first_pos + 256 k - 1 and 256 k
    for k in (6, 7):
        for d in (-1, 0, -1, 0):
            R.add(tile(k) + d, "60M", lib=d % 3)
    # 40 leading reads that end before the last warp's window [pos0 + 224, pos0 + 256), then reads covering it
    t8 = tile(8)
    for k in range(40):
        R.add(t8 + k, "20M", lib=k % 3)
    for k in range(12):
        R.add(t8 + 200 + k, "40M", lib=k % 3)
    # CIGAR ops per 96-read chunk: 188 (a 4-aligned window of at most 192 whatever the chunk's first op index) and 195 (> 192)
    for t, cig in ((9, "50M"), (10, "3S40M2S")):
        for k in range(96):
            R.add(tile(t) + 10 + 2 * k, cig if k < 4 - (t == 10) else "5S45M", lib=k % 3)
    c = _case("chunks", ref, R.build(), [(0, 1, L)], n_libs=3,
              targets=["chunk_reads", "hot_run_end", "warp_edges", "tile_edges", "lead_skip", "libless_hot", "cigar_stage"])
    # the K1 tiles (TILE sites from first_pos = 0) each edge target was built in
    c["probe"] = dict(warp_tile=10, warp_windows=(1, 3, 6), edge_tiles=(12, 14), lead_tile=16, libless_tile=8)
    return c


def narrow_escape(seed=405):
    """Sites covered by 254, 255 and 256 reads (some dead: npass < ncover); clipped-length sums of exactly 65 535 and 65 536;
    SE-mapq sums around 65 535 from SM tags and a negative SM; a mismatch-quality sum of 65 535 and 65 536."""
    L = 6000
    ref = _ref(seed, L)
    R = _Reads(ref, seed)
    ok_q = lambda n: np.full(n, 30, np.uint8)

    def stack(p, n, cig, **kw):
        for k in range(n):
            R.add(p, cig, qual=ok_q(sum(l for l, o in _ops(cig) if o in "MIS=X")), sub_rate=0.0,
                  flag=kw.get("flag", 0 if k % 3 else 16) | (1024 if k % 17 == 5 else 0), lib=kw.get("lib", 0), nm=1,
                  sm=kw.get("sm"), q2_tail=False)
    # depth 254 / 255 / 256 (dead duplicates among them)
    stack(200, 254, "30M")
    R.add(203, "30M", qual=ok_q(30), sub_rate=0.0, flag=0, lib=0)
    R.add(206, "30M", qual=ok_q(30), sub_rate=0.0, flag=0, lib=0)
    # clip sums: 255 x 257 = 65535 and 254 x 257 + 258 = 65536 (every read passing, same base)
    for p, last in ((600, 257), (1200, 258)):
        for k in range(255):
            lq = last if k == 254 else 257
            R.add(p, f"{lq}M", qual=ok_q(lq), sub_rate=0.0, flag=0 if k % 2 else 16, lib=0, q2_tail=False)
    # SE-mapq sums from SM (proper pairs): 255 x 257 = 65535, + 1 -> 65536, and a negative SM
    for p, extra in ((2000, 0), (2100, 1), (2200, -300)):
        for k in range(255):
            sm = 257 + (extra if k == 254 else 0)
            R.add(p, "40M", qual=ok_q(40), sub_rate=0.0, flag=3, lib=1, sm=sm if extra >= 0 or k != 254 else -5, q2_tail=False)
    R.add(2235, "40M", qual=ok_q(40), sub_rate=0.0, flag=3, lib=1, sm=-5, q2_tail=False)   # alone past the stack: the sum wraps
    # mismatch-quality sums: 7 isolated mismatches per read with qualities 40 x 6 + 17 = 257 (258 in one read)
    for p, last in ((3000, 257), (3400, 258)):
        span = 80
        for k in range(255):
            seq = list(edge_cases._read_from_ref(R.rng, ref, p, [(span, "M")], 0.0))
            q = np.full(span, 35, np.uint8)
            for j, off in enumerate((5, 15, 25, 35, 45, 55, 65)):
                seq[off] = {"A": "C", "C": "G", "G": "T", "T": "A"}[seq[off]]
                q[off] = 40 if j < 6 else (17 + (last - 257 if k == 254 else 0))
            R.add(p, f"{span}M", seq="".join(seq), qual=q, flag=0, lib=2, q2_tail=False)
    sites = [203, 205, 206, 210, 700, 1300, 2010, 2110, 2210, 3010, 3410]
    regions = [(0, 1, L)] + [(0, s + 1, s + 1) for s in sites]
    return _case("narrow", ref, R.build(), regions, n_libs=3, targets=["ncover_8bit", "clip_sum_16bit", "se_sum_16bit", "mmq_sum_16bit"])


def deep_kernel(seed=406):
    """Single-site tiles under 255, 256 and 257 reads (deep_site_kernel blocks of 256); groups with 8 and 9 distinct insertion
    alleles (DEEP_ICACHE = 8); insertions of 8 and 9 bases and deletions of 127 and 128 bases (the cacheable limits)."""
    L = 5000
    ref = _ref(seed, L)
    R = _Reads(ref, seed)
    for s, n in ((300, 255), (700, 256), (1100, 257)):
        for k in range(n):
            R.add(s - int(R.rng.integers(0, 40)), "60M", lib=k % 3, sub_rate=0.03, flag=1024 if k % 29 == 3 else None)
    alleles = ["A", "C", "G", "T", "AC", "CG", "GT", "TA", "ACG"]
    for s, n_al in ((1600, 8), (2000, 9)):
        for k in range(80):
            a = alleles[k % n_al]
            p = s - 20
            body = edge_cases._read_from_ref(R.rng, ref, p, [(21, "M")], 0.01) + a + \
                edge_cases._read_from_ref(R.rng, ref, s + 1, [(30, "M")], 0.01)
            R.add(p, f"21M{len(a)}I30M", seq=body, lib=k % 3)
    for s, kind, ln in ((2600, "I", 8), (2610, "I", 9), (3000, "D", 127), (3400, "D", 128)):
        for k in range(30):
            p = s - 20
            if kind == "I":
                ins = "".join("ACGT"[int(x)] for x in R.rng.integers(0, 4, ln)) if k % 3 == 0 else "ACGTTGCA" + "C" * (ln - 8)
                body = edge_cases._read_from_ref(R.rng, ref, p, [(21, "M")], 0.01) + ins + \
                    edge_cases._read_from_ref(R.rng, ref, s + 1, [(30, "M")], 0.01)
                R.add(p, f"21M{ln}I30M", seq=body, lib=k % 3)
            else:
                R.add(p, f"21M{ln if k % 4 else ln - 1}D30M", lib=k % 3)
    sites = [300, 700, 1100, 1600, 2000, 2600, 2610, 3000, 3400]
    regions = [(0, s + 1, s + 1) for s in sites] + [(0, 2590, 2640)]
    return _case("deep", ref, R.build(), regions, n_libs=3, targets=["deep_block", "icache", "indel_len"])


def byte_values(seed=407):
    """Reads with QUAL '*' (every quality byte 0xFF) and MAPQ 255 mixed with ordinary reads."""
    L = 3000
    ref = _ref(seed, L)
    R = _Reads(ref, seed)
    for k in range(400):
        p = 100 + 6 * k
        r = k % 5
        if r == 0:
            R.add(p, "70M", qual=np.full(70, 0xFF, np.uint8), lib=k % 2, sub_rate=0.05)
        elif r == 1:
            R.add(p, "4S66M", mapq=255, lib=k % 2, sub_rate=0.05)
        elif r == 2:
            R.add(p, "30M2I38M", qual=np.full(70, 0xFF, np.uint8), mapq=255, lib=k % 2, sub_rate=0.05)
        else:
            R.add(p, "70M", mapq=int(R.rng.choice([60, 19, 20])), lib=k % 2, sub_rate=0.05)
    return _case("values", ref, R.build(), [(0, 1, L)], n_libs=2, targets=["byte_values"])


def queue_rows(seed=408):
    """-p with 40 libraries over argv regions, adjacent and overlapping.  Library rows >= SEL_LAST_ROWS (32) hold deletions
    anchored at the last site of a region that no lower row covers and whose line shows no alternative allele: the deletion prints
    only in the next region, from the never-cleared deletion queue, so the site selection must ship that site for those rows.
    Rows < 32 do the same at the end of a later region (sel_site_kernel's shared-memory branch).

    Not part of all_cases(): the reference prints -p library blocks in the order of the library NAMES, and the SAM of a case names
    library k "lib<k>", so with more than ten libraries its block order (lib0, lib1, lib10, ...) is not the row order the oracle
    and the engine print.  The engine is compared with the oracle on it."""
    L = 3000
    ref = _ref(seed, L)
    R = _Reads(ref, seed)
    for end0, rows in ((1099, range(32, 40)), (1399, range(33, 40, 2)), (1699, range(0, 8)), (1999, range(30, 36))):
        for k, r in enumerate(rows):
            R.add(end0 - 29, f"30M{3 + (k % 2)}D30M", lib=r, sub_rate=0.0, q2_tail=False)
        for k in range(24):     # the region's inner sites, from other rows, ending before its last site
            R.add(end0 - 95 + 2 * k, "40M", lib=(k * 7) % 40 if end0 != 1099 else k % 30, sub_rate=0.03)
    for k in range(30):         # library-less reads away from the probed sites
        R.add(2300 + 10 * k, "50M", lib=None if k % 5 == 0 else k % 40, sub_rate=0.03)
    regions = [(0, 1001, 1100), (0, 1101, 1200), (0, 1301, 1400), (0, 1391, 1450), (0, 1601, 1700), (0, 1701, 1750),
               (0, 1901, 2000), (0, 1995, 2100), (0, 2290, 2700)]
    c = _case("queue_rows", ref, R.build(), regions, site_list=False, modes=(False,), n_libs=40, targets=["queue_rows"])
    c["probe"] = dict(anchors=(1099, 1399), low_anchors=(1699,))   # 0-based region ends: deletions only from rows >= 32 / < 32
    return c


# the flag sets every boundary case runs with
FLAG_SETS = {
    "default": dict(),
    "q20b20": dict(min_mapq=20, min_bq=20),
    "perlib": dict(per_lib=True),
    "ic": dict(insertion_centric=True),
    "perlib_ic_q20b20": dict(per_lib=True, insertion_centric=True, min_mapq=20, min_bq=20),
    "d": dict(max_cnt=200),
}


@functools.lru_cache(maxsize=None)
def all_cases():
    return (length_ladder(), clip_numerators(),
            ref_window(0, 16000, 411), ref_window(1, 16001, 412), ref_window(4095, 20002, 413), ref_window(4097, 20003, 414),
            chunk_geometry(), narrow_escape(), deep_kernel(), byte_values())


def jobs():
    """(case, flag-set name, flags, site_list mode, key) for every run the anchor and the engine comparison make."""
    out = []
    for c in all_cases():
        for fname, fl in FLAG_SETS.items():
            for sl in c["modes"]:
                out.append((c, fname, fl, sl, f"{c['name']}_{fname}_{'l' if sl else 'argv'}"))
    return out
