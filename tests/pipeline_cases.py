"""Cases for the pipelined push path and the pools at production scale (tests/test_pipeline_scale.py).

compute_pipelined (csrc/brc_engine.cu) cuts a borrowed single-region batch into read-index chunks: chunk c holds reads
[n c / N, n (c + 1) / N), and after its K0 the pileup kernel runs on the tiles that end at or before the first position of
chunk c + 1.  The builders here place reads so that those cuts land where that rule has edges; `pipe_plan` restates the rule
and `cut_kinds` names the edges a chunk count reaches, so a test can assert that they were reached.

Every case is a dict in the tests/cases.py shape.  Deterministic: every builder takes its own seed."""
from __future__ import annotations

import functools

import numpy as np

from boundary_cases import K1_TILE, _case, _ref, _Reads

TILE = K1_TILE
# chunk counts of the cut tests.  A run cuts its own input into at most 32 chunks; every pileup launch takes a tile dispenser of
# its own.  65: a 65th one; 200: enough chunks that finish a tile for the chunk-cut case to make more than 64 pileup launches in one run.
CHUNK_COUNTS = (1, 2, 3, 7, 32, 64, 65, 200)
CUT_KINDS = ("in_run", "on_edge", "off_edge", "before_region", "no_tile", "later_tile")
_CIGARS = ("100M", "100M", "100M", "48M3D52M", "30M2I68M", "5S95M", "90M10S", "60M1D40M")
_CIGARS150 = ("150M", "150M", "150M", "98M3D52M", "30M2I118M", "5S145M", "140M10S", "110M1D40M")


def pipe_plan(pos, first_pos: int, n_tiles: int, n_chunks: int):
    """compute_pipelined's chunk loop restated: per chunk (a, b, tile_from, tile_to).  Reads [a, b) go through K0; the pileup
    kernel runs on tiles [tile_from, tile_to) when that range is not empty."""
    n = len(pos)
    n_chunks = max(1, min(n_chunks, n))
    out, done = [], 0
    for c in range(n_chunks):
        a, b = n * c // n_chunks, n * (c + 1) // n_chunks
        if c + 1 < n_chunks:
            nxt = int(pos[b])
            to = 0 if nxt <= first_pos else min(n_tiles, (nxt - first_pos) // TILE)
            to = max(to, done)
        else:
            to = n_tiles
        out.append((a, b, done, to))
        done = max(done, to)
    return out


def pipe_launches(plan, n_deep: int = 0, selection_kernels: int = 0) -> int:
    """brc_last_launch_count after compute_pipelined: init, one K0 per chunk, one pileup (and one deep-site) launch per chunk
    that finishes tiles, the selection kernels."""
    k1 = sum(1 for _, _, t0, t1 in plan if t1 > t0)
    return 1 + len(plan) + k1 * (2 if n_deep else 1) + selection_kernels


def cut_kinds(pos, first_pos: int, n_tiles: int, n_chunks: int) -> set:
    """Which edges of the chunk rule the cuts of `n_chunks` chunks reach:
      in_run         the cut falls between two reads at the same position
      on_edge        the next chunk's first read starts exactly on a tile edge (first_pos + 256 k, k > 0)
      off_edge       ... one position before or after one
      before_region  ... at or before first_pos (reads that start before the region: no tile is finished)
      no_tile        a chunk other than the last finishes no tile (no pileup launch)
      later_tile     every read of a chunk starts in a tile that chunk does not finish"""
    kinds = set()
    plan = pipe_plan(pos, first_pos, n_tiles, n_chunks)
    for a, b, t0, t1 in plan[:-1]:
        p, q = int(pos[b - 1]), int(pos[b])
        if p == q:
            kinds.add("in_run")
        if q <= first_pos:
            kinds.add("before_region")
        elif (q - first_pos) % TILE == 0:
            kinds.add("on_edge")
        elif (q - first_pos) % TILE in (1, TILE - 1):
            kinds.add("off_edge")
        if t1 == t0:
            kinds.add("no_tile")
        if t1 > 0 and int(pos[a]) > first_pos and (int(pos[a]) - first_pos) // TILE >= t1:
            kinds.add("later_tile")
    return kinds


def _positions(rng, first_pos):
    """Read start positions, sorted: a lead-in of reads starting before the region, even coverage, a run of 300 reads at one
    position, a gap of 4 kb where no read starts, a dense stretch of 600 reads within 200 bp, even coverage again."""
    seg = [np.sort(rng.integers(first_pos - 80, first_pos + 1, 150)),
           np.arange(first_pos + 1, 9000, 8) + rng.integers(0, 4, len(range(first_pos + 1, 9000, 8))),
           np.full(300, 9100),
           np.arange(9101, 12000, 8),
           np.sort(rng.integers(16000, 16200, 600)),
           np.arange(16200, 29000, 8)]
    p = np.sort(np.concatenate(seg)).astype(np.int64)
    n = p.shape[0]
    # the cuts of 2 and 3 chunks on a tile edge, one past one and one before one
    for b, d in ((n // 2, 0), (n // 3, 1), (2 * n // 3, -1)):
        edge = first_pos + TILE * int(round((int(p[b]) - first_pos) / TILE)) + d
        p[b] = edge
        p[:b] = np.minimum(p[:b], edge)
        p[b + 1:] = np.maximum(p[b + 1:], edge)
    return p


@functools.lru_cache(maxsize=None)
def chunk_cuts(n_libs: int = 3, seed: int = 501):
    """One argv region (beg 2001: first_pos 1999) over 29 kb whose read positions put the cuts of CHUNK_COUNTS on every edge of
    the chunk rule (cut_kinds).  Reads carry indels, clips, 2 % substitutions and mixed MAPQ; library ids cycle over n_libs.
    Library k is named "lib%02d" so that name order is row order for the reference binary's -p blocks."""
    L = 30000
    first_pos = 1999
    ref = _ref(seed, L)
    R = _Reads(ref, seed)
    pos = _positions(np.random.default_rng(seed), first_pos)
    for k, p in enumerate(pos):
        cig = _CIGARS[int(R.rng.integers(0, len(_CIGARS)))]
        R.add(int(p), cig, mapq=int(R.rng.choice([60, 60, 60, 30, 15, 0])), lib=k % n_libs, sub_rate=0.02)
    c = _case(f"cuts{n_libs}", ref, R.build(), [(0, first_pos + 2, L)], site_list=False, modes=(False,), n_libs=n_libs)
    return c


@functools.lru_cache(maxsize=None)
def carried_regions(seed: int = 501):
    """chunk_cuts' reads over four argv regions, adjacent and overlapping, for the carried deletion queue (one brc_compute per
    region, each region's reads one borrowed push)."""
    c = chunk_cuts(3, seed)
    return dict(c, name="cuts_carry", regions=[(0, 2001, 9100), (0, 9101, 12500), (0, 12400, 20000), (0, 20001, 29100)])


@functools.lru_cache(maxsize=None)
def deep_site(seed: int = 502, depth: int = 2500):
    """One site-list line, one site under `depth` reads (>= the deep-site kernel's 2048): its tile goes to deep_site_kernel."""
    L = 3000
    s = 1000
    ref = _ref(seed, L)
    R = _Reads(ref, seed)
    for k, p in enumerate(np.sort(R.rng.integers(s - 99, s + 1, depth))):
        R.add(int(p), _CIGARS[k % len(_CIGARS)], mapq=int(R.rng.choice([60, 60, 20, 0])), lib=k % 3, sub_rate=0.03)
    c = _case("deep_site", ref, R.build(), [(0, s + 1, s + 1)], site_list=True, modes=(True,), n_libs=3)
    return c


LONG_READS = (16000, 25000, 16001)


@functools.lru_cache(maxsize=None)
def offsets(seed: int = 503):
    """About 5000 reads of 150 bp every 10 bp over 50 kb, with three reads of 16-25 kb among them: a K0 block or K1 chunk holding
    one of those is never staged in shared memory, so their bytes are read from the pools with full offsets."""
    L = 60000
    ref = _ref(seed, L)
    R = _Reads(ref, seed)
    for k, p in enumerate(range(100, 50000, 10)):
        R.add(p, _CIGARS150[k % len(_CIGARS150)], mapq=int(R.rng.choice([60, 60, 30])), lib=k % 3, sub_rate=0.02)
    for p, lq in zip((20003, 30007, 40011), LONG_READS):
        R.add(p, f"{lq // 2}M2D{lq - lq // 2}M", lib=1, sub_rate=0.01)
    c = _case("offsets", ref, R.build(), [(0, 1, L)], site_list=True, modes=(True,), n_libs=3)
    return c


def jobs():
    """(case, flag-set name, flags, site_list mode, key) for every case of this module the reference binary is run on.  Not
    chunk_cuts(12): the SAM of a case names library k "lib<k>", and with more than ten libraries the reference prints its -p
    blocks in name order (lib0, lib1, lib10, ...), not in the row order the oracle and the engine print; the engine is compared
    with the oracle on it."""
    import cases
    out = []
    for fname, fl in cases.FLAG_SETS.items():
        out.append((chunk_cuts(3), fname, fl, False, f"cuts3_{fname}"))
    for fname in ("default", "perlib"):
        out.append((carried_regions(), fname, cases.FLAG_SETS[fname], False, f"carry_{fname}"))
        out.append((deep_site(), fname, cases.FLAG_SETS[fname], True, f"deep_site_{fname}"))
        out.append((offsets(), fname, cases.FLAG_SETS[fname], True, f"offsets_{fname}"))
    return out
