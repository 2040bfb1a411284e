"""The pipelined push path, the persistent pileup grid and the byte pools at production shapes, bit for bit against the oracle.

Cases: tests/pipeline_cases.py.  BRC_PIPE_CHUNKS (read on every brc_compute) sets how many read-index chunks compute_pipelined
cuts a borrowed batch into; pipeline_cases.pipe_plan restates that loop, so each test knows which launches the run must make.

CPU
  audit    the cut positions of every chunk count reach every edge of the chunk rule (pipeline_cases.cut_kinds); 200 chunks make
           more than 64 pileup launches; the pool-offset runs straddle 2^31 / 2^32 where they claim to.
  anchor   the oracle's text on every new case and flag set against the SHA-256 of what the unmodified reference binary printed
           (tests/golden/pipeline_sha256.json, written by tests/golden/make_golden.py --pipeline-only).
GPU, each asserting that it reached its path
  test_chunk_cuts_equal_the_oracle           every chunk count x cases.FLAG_SETS: K0 per chunk, the pileup kernel on the
                                             tiles a chunk finishes, per-chunk word copies at s0 > 0, pool records shipped
                                             in pieces, a tile dispenser for each of more than 64 launches.  Launch count = plan.
  test_multi_chunk_per_library_rows          -p with 3 rows (per-array copies) and 12 rows (one strided 2-D copy at s0 > 0).
  test_multi_chunk_site_filter               the site selection after a chunked run (no per-chunk copies).
  test_multi_chunk_pool_overflow_falls_back  compute_pipelined overflows its pool and the plain path recomputes.
  test_multi_chunk_deep_site                 the deep-site kernel launched from the chunk loop.
  test_multi_chunk_carried_queue             brc_set_queue_carry, one brc_compute per argv region, several chunks each.
  test_starved_pileup_grid                   one CTA per SM (BRC_K1_RESERVE_CTAS, in a fresh process) on more tiles than CTAs,
                                             on the plain path and in every pileup launch of 2 and 3 chunks.
  test_device_pools_past_2_31_and_2_32       brc_run_device with quality or base pools whose offsets cross 2^31 / 2^32."""
import functools
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import cases
import pipeline_cases as pc
from cases import ROOT, first_diff, region_geometry

CSRC = os.path.join(ROOT, "bam_readcount_b200", "csrc")


@functools.lru_cache(maxsize=None)
def _select_kernels() -> int:
    src = open(os.path.join(CSRC, "brc_device.cuh")).read()
    return int(re.search(r"constexpr\s+int\s+SELECT_KERNELS\s*=\s*(\d+);", src).group(1))


def _plan(case, n_chunks, region=None):
    _, _, _, sub, first_pos, _, n_tiles = region_geometry(case, region or case["regions"][0])
    return pc.pipe_plan(sub.pos, first_pos, n_tiles, n_chunks)


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
def test_chunk_cuts_reach_every_edge_of_the_chunk_rule():
    for n_libs in (3, 12):
        case = pc.chunk_cuts(n_libs)
        _, _, _, sub, first_pos, n_slots, n_tiles = region_geometry(case, case["regions"][0])
        assert sub.n_reads == case["batch"].n_reads
        reached = set()
        for n in pc.CHUNK_COUNTS:
            reached |= pc.cut_kinds(sub.pos, first_pos, n_tiles, n)
        assert reached == set(pc.CUT_KINDS), set(pc.CUT_KINDS) - reached
        # the cuts of 2 and 3 chunks sit on a tile edge, one after one and one before one
        assert {"on_edge"} <= pc.cut_kinds(sub.pos, first_pos, n_tiles, 2) and {"off_edge"} <= pc.cut_kinds(sub.pos, first_pos, n_tiles, 3)
        # no tile of <= 2 sites: no deep-site tile, so the launch count of a plan is 1 + chunks + pileup launches
        assert n_slots % pc.TILE > 2
        k1 = {n: sum(1 for _, _, t0, t1 in pc.pipe_plan(sub.pos, first_pos, n_tiles, n) if t1 > t0) for n in pc.CHUNK_COUNTS}
        assert k1[200] > 64, k1                     # every pileup launch of a run has its own tile dispenser, the 65th and later ones too
        assert all(k1[n] > 1 for n in pc.CHUNK_COUNTS if n > 1), k1
    carry = pc.carried_regions()
    for region in carry["regions"]:
        _, _, _, sub, first_pos, n_slots, n_tiles = region_geometry(carry, region)
        assert sub.n_reads < 2048 and sum(1 for _, _, t0, t1 in pc.pipe_plan(sub.pos, first_pos, n_tiles, 7) if t1 > t0) > 1


def test_deep_site_case_takes_the_deep_kernel():
    case = pc.deep_site()
    _, _, _, sub, first_pos, n_slots, n_tiles = region_geometry(case, case["regions"][0])
    assert sub.n_reads >= 2048 and n_slots <= 2 and n_tiles == 1


JOBS = pc.jobs()


@pytest.mark.parametrize("job", JOBS, ids=[j[4] for j in JOBS])
def test_oracle_equals_reference_binary_on_pipeline_cases(job):
    case, fname, fl, sl, key = job
    cases.assert_anchor("pipeline_sha256.json", key, cases.run_oracle(case, fl, site_list=sl).text)


# ---------------------------------------------------------------------------------------------------------------------------
# GPU: chunked push path
# ---------------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _one_chunk_text(fname):
    old = os.environ.get("BRC_PIPE_CHUNKS")
    os.environ["BRC_PIPE_CHUNKS"] = "1"
    try:
        return cases.run_engine(pc.chunk_cuts(3), cases.FLAG_SETS[fname], False, dump=False).text
    finally:
        if old is None:
            del os.environ["BRC_PIPE_CHUNKS"]
        else:
            os.environ["BRC_PIPE_CHUNKS"] = old


@pytest.mark.gpu
@pytest.mark.parametrize("n_chunks", pc.CHUNK_COUNTS)
def test_chunk_cuts_equal_the_oracle(n_chunks, monkeypatch):
    """Every chunk count on chunk_cuts(3), every flag set: raw accumulators, text and warning counters equal the oracle's, the
    text equals the one-chunk run's, and the launch count is the plan's (so the run was cut into that many chunks).  -d 5 is
    below the batch size, so that batch is copied and takes the plain path: three launches."""
    case = pc.chunk_cuts(3)
    plan = _plan(case, n_chunks)
    for fname, fl in cases.FLAG_SETS.items():
        want = cases.run_oracle_cached(case, fl, False)
        one = _one_chunk_text(fname)
        monkeypatch.setenv("BRC_PIPE_CHUNKS", str(n_chunks))
        got = cases.run_engine(case, fl, False)
        cases.assert_same(got, want, f"{n_chunks} chunks, {fname}")
        assert got.text == one, f"{n_chunks} chunks, {fname}: text differs from one chunk"
        assert got.launches == (3 if "max_cnt" in fl else pc.pipe_launches(plan)), (fname, got.launches)
    if n_chunks > 1:                # word copies of later chunks start past slot 0; pool records leave in pieces
        assert any(t0 > 0 and t1 > t0 for _, _, t0, t1 in plan) and got.n_sec > 0


@pytest.mark.gpu
@pytest.mark.parametrize("n_libs", [3, 12])
@pytest.mark.parametrize("n_chunks", [7, 65])
def test_multi_chunk_per_library_rows(n_libs, n_chunks, monkeypatch):
    """-p: 3 rows x 8 words take one plain copy per array of each chunk's finished slots; 12 rows x 8 words (> 64 arrays) take
    one strided 2-D copy, at s0 > 0 from the second pileup launch on."""
    case = pc.chunk_cuts(n_libs)
    assert (n_libs * 8 > 64) == (n_libs == 12)
    plan = _plan(case, n_chunks)
    monkeypatch.setenv("BRC_PIPE_CHUNKS", str(n_chunks))
    for fname in ("perlib", "perlib_ic_q20b20"):
        fl = cases.FLAG_SETS[fname]
        got = cases.run_engine(case, fl, False)
        cases.assert_same(got, cases.run_oracle(case, fl, site_list=False), f"{n_libs} libraries, {n_chunks} chunks, {fname}")
        assert got.launches == pc.pipe_launches(plan)


@pytest.mark.gpu
@pytest.mark.parametrize("n_chunks", [7, 65])
def test_multi_chunk_site_filter(n_chunks, monkeypatch):
    """With a site filter, the chunk loop skips the per-chunk copies and the selection kernels run after it: the filtered text is
    select_lines (tests/site_filter_rule.py) of the oracle's."""
    from site_filter_rule import THRESHOLDS, select_lines
    case = pc.chunk_cuts(3)
    plan = _plan(case, n_chunks)
    monkeypatch.setenv("BRC_PIPE_CHUNKS", str(n_chunks))
    for fname in ("default", "perlib"):
        otext = cases.run_oracle_cached(case, cases.FLAG_SETS[fname], False).text
        for mc, mf in THRESHOLDS:
            got = cases.run_engine(case, cases.FLAG_SETS[fname], False, site_filter=(mc, mf))
            want = select_lines(otext, mc, mf)
            assert got.text == want, (fname, mc, mf, first_diff(got.text, want))
            assert got.launches == pc.pipe_launches(plan, selection_kernels=_select_kernels()), (fname, got.launches)


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [dict(), dict(per_lib=True)], ids=["alllib", "perlib"])
@pytest.mark.parametrize("n_chunks", [7, 65])
def test_multi_chunk_pool_overflow_falls_back(flags, n_chunks, monkeypatch):
    """boundary_cases.pool_case (random bases: four or five base classes per site) in many chunks: compute_pipelined's pool
    overflows, brc_compute falls back to the plain path, which grows the pool.  The fallback shows in the launch count (the plain
    path's three, not the chunk plan's) and in a pool larger than its initial capacity."""
    from boundary_cases import initial_pool_cap, pool_case
    case = pool_case()
    plan = _plan(case, n_chunks)
    assert pc.pipe_launches(plan) > 3 + n_chunks
    monkeypatch.setenv("BRC_PIPE_CHUNKS", str(n_chunks))
    got = cases.run_engine(case, flags, True)
    cases.assert_same(got, cases.run_oracle(case, flags, site_list=True), f"{n_chunks} chunks")
    assert got.launches == 3, f"launch count {got.launches}: the pipelined run did not fall back"
    n_slots = region_geometry(case, case["regions"][0])[5]
    assert got.n_sec > initial_pool_cap(case, flags, n_slots)


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [dict(), dict(per_lib=True)], ids=["alllib", "perlib"])
@pytest.mark.parametrize("n_chunks", [7, 65])
def test_multi_chunk_deep_site(flags, n_chunks, monkeypatch):
    """One site-list site under 2453 reads: its one tile is finished by the last chunk, whose pileup launch is followed by the
    deep-site kernel (the launch count holds both)."""
    case = pc.deep_site()
    plan = _plan(case, n_chunks)
    assert len(plan) == n_chunks and sum(1 for _, _, t0, t1 in plan if t1 > t0) == 1
    monkeypatch.setenv("BRC_PIPE_CHUNKS", str(n_chunks))
    got = cases.run_engine(case, flags, True)
    cases.assert_same(got, cases.run_oracle(case, flags, site_list=True), f"{n_chunks} chunks")
    assert got.launches == pc.pipe_launches(plan, n_deep=1), got.launches


@pytest.mark.gpu
@pytest.mark.parametrize("fname", ["default", "perlib"])
def test_multi_chunk_carried_queue(fname, monkeypatch):
    """brc_set_queue_carry on: four adjacent and overlapping argv regions, one brc_compute each, each region's reads one borrowed
    push in 7 chunks.  The concatenated text equals the four regions as one batch, and the oracle's."""
    case = pc.carried_regions()
    fl = cases.FLAG_SETS[fname]
    otext = cases.run_oracle_cached(case, fl, False).text
    one = cases.run_engine(case, fl, False).text
    assert one == otext, first_diff(one, otext)
    monkeypatch.setenv("BRC_PIPE_CHUNKS", "7")
    runs = cases.run_engine_per_region(case, fl, False)
    for region, r in zip(case["regions"], runs):
        assert r.launches == pc.pipe_launches(_plan(case, 7, region)), region
    parts = "".join(r.text for r in runs)
    assert parts == one, first_diff(parts, one)


# ---------------------------------------------------------------------------------------------------------------------------
# GPU: one CTA per SM
# ---------------------------------------------------------------------------------------------------------------------------
def _starved_jobs():
    import boundary_cases
    from boundary_cases import pool_case, selection_cases
    big = selection_cases()[0]
    big = dict(big, regions=big["regions"][:1])               # one argv region of 300 000 sites
    jobs = [("300k_sites", big, dict(), False, 0), ("pool_perlib", pool_case(), dict(per_lib=True), True, 0),
            ("chunk_geometry", boundary_cases.chunk_geometry(), dict(per_lib=True), True, 0),
            ("chunk_geometry_alllib", boundary_cases.chunk_geometry(), dict(), True, 0)]
    # the chunked push path on the same starved grid: every pileup launch of these plans has several tiles per CTA
    for n_chunks in (2, 3):
        jobs += [(f"300k_sites_chunks{n_chunks}", big, dict(), False, n_chunks),
                 (f"300k_sites_perlib_chunks{n_chunks}", big, dict(per_lib=True), False, n_chunks)]
    return jobs


def starved_child():
    """Runs in a fresh process with BRC_K1_RESERVE_CTAS set (launch_pileup reads it once per process): each job's dump, text and
    warnings against the oracle, and for the chunked jobs (BRC_PIPE_CHUNKS) the launch count; prints one JSON line."""
    out = {}
    for name, case, flags, sl, n_chunks in _starved_jobs():
        want = cases.run_oracle(case, flags, site_list=sl)
        if n_chunks:
            os.environ["BRC_PIPE_CHUNKS"] = str(n_chunks)
        try:
            got = cases.run_engine(case, flags, site_list=sl)
        finally:
            os.environ.pop("BRC_PIPE_CHUNKS", None)
        w = got.warnings
        out[name] = dict(dump=got.dump == want.dump, text=got.text == want.text, warn=[w[0], w[1], w[3]] == list(want.warnings),
                         launches=got.launches if n_chunks else 0, diff=first_diff(got.dump, want.dump))
    print("STARVED " + json.dumps(out))


@pytest.mark.gpu
def test_starved_pileup_grid():
    """BRC_K1_RESERVE_CTAS larger than every CTA slot drops the pileup grid to its floor of one CTA per SM, so every CTA takes
    many tiles from the dispenser and carries site_reset, its shared second-class cells, the stage ring's parity and its warning
    slots from one tile to the next (the 300 000-site region: 1172 tiles on 132 CTAs of an H100).  That region without -p, the
    random-base pool case and chunk_geometry (each fewer work items than SMs: one CTA per item under the same grid rule) equal
    the oracle.  The 300 000-site region also runs through the chunked push path at 2 and 3 chunks, with and without -p: every
    pileup launch of those plans has more than two tiles per CTA, so each CTA takes several tiles inside one chunk's launch, and
    the launch count is the plan's."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    reserve = 1 << 20
    grid = max(3 * sms - reserve, sms)                        # launch_pileup: max(SMs x BRC_K1_CTAS_PER_SM - reserve, SMs)
    big = _starved_jobs()[0][1]
    n_tiles = region_geometry(big, big["regions"][0])[6]
    assert n_tiles > 8 * grid, (n_tiles, grid)               # 300 000 sites: every CTA takes at least eight tiles
    plans = {n: _plan(big, n) for n in (2, 3)}
    for n, plan in plans.items():
        k1 = [t1 - t0 for _, _, t0, t1 in plan if t1 > t0]
        assert len(k1) == n and min(k1) > 2 * grid, (n, k1, grid)
    env = dict(os.environ, BRC_K1_RESERVE_CTAS=str(reserve))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-c", f"import sys; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]; import test_pipeline_scale as t; t.starved_child()"]
    p = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-3000:]
    line = [ln for ln in p.stdout.splitlines() if ln.startswith("STARVED ")]
    assert line, p.stdout[-2000:]
    res = json.loads(line[-1][len("STARVED "):])
    assert set(res) == {j[0] for j in _starved_jobs()}
    for name, case, flags, sl, n_chunks in _starved_jobs():
        r = res[name]
        assert r["dump"] and r["text"] and r["warn"], (name, r)
        if n_chunks:
            assert r["launches"] == pc.pipe_launches(plans[n_chunks]), (name, r["launches"])


# ---------------------------------------------------------------------------------------------------------------------------
# GPU: pools past 2^31 and 2^32 bytes
# ---------------------------------------------------------------------------------------------------------------------------
def _deltas(sub, pool):
    """δ per run: the bytes of the pool before the boundary.  'staged': the boundary falls inside read 40, which sits in a K0 block
    and a K1 chunk that are both staged; 'long': inside the first read too long for any stage."""
    off = (sub.qual_off if pool == "qual" else sub.seq_off).astype(np.int64)
    j = int(np.nonzero(sub.l_qseq >= 16000)[0][0])
    return dict(staged=int(off[40] + (off[41] - off[40]) // 2), long=int(off[j] + (off[j + 1] - off[j]) // 2))


def _straddles(sub, pool, lead, bound, first_pos, n_slots):
    """What the kernels will do around the boundary with the pool shifted by `lead`: (a staged K0 block straddles it, a staged K1
    chunk straddles it, an unstaged read straddles it)."""
    import dataclasses
    from kernel_model import k1_chunks, kernel_constants, tile_ranges
    K = kernel_constants()
    key = "qual_off" if pool == "qual" else "seq_off"
    b = dataclasses.replace(sub, **{key: sub.__dict__[key].astype(np.uint64) + np.uint64(lead)})
    qo, so = b.qual_off.astype(np.int64), b.seq_off.astype(np.int64)
    off = qo if pool == "qual" else so
    n = b.n_reads
    k0, k0_staged = False, []
    for r0 in range(0, n, K["K0_READS"]):
        r1 = min(n, r0 + K["K0_READS"])
        qa, qb, sa, sb = qo[r0] & ~15, (qo[r1] + 15) & ~15, so[r0] & ~15, (so[r1] + 15) & ~15
        a, z = (qa, qb) if pool == "qual" else (sa, sb)
        k0_staged.append(bool(qb - qa <= K["K0_QUAL_CAP"] and sb - sa <= K["K0_SEQ_CAP"]))
        k0 |= k0_staged[-1] and bool(a < bound < z)
    k1 = any(c["staged"] and off[c["r0"]] < bound < off[c["r1"]] for c in k1_chunks(b, tile_ranges(b, first_pos, first_pos + n_slots)))
    # a read whose qualities alone overflow K1's stage, in an unstaged K0 block
    long_read = any(off[i] < bound < off[i + 1] and b.l_qseq[i] + 32 > K["STAGE_QUAL"] and not k0_staged[i // K["K0_READS"]]
                    for i in range(n))
    return k0, k1, long_read


def test_pool_offset_runs_straddle_their_boundaries():
    case = pc.offsets()
    _, _, _, sub, first_pos, n_slots, _ = region_geometry(case, case["regions"][0])
    for pool in ("qual", "seq"):
        for bound in (1 << 31, 1 << 32):
            d = _deltas(sub, pool)
            assert _straddles(sub, pool, bound - d["staged"], bound, first_pos, n_slots)[:2] == (True, True), (pool, bound)
            assert _straddles(sub, pool, bound - d["long"], bound, first_pos, n_slots)[2], (pool, bound)


@pytest.mark.gpu
@pytest.mark.parametrize("bound", [1 << 31, 1 << 32], ids=["2^31", "2^32"])
@pytest.mark.parametrize("pool", ["qual", "seq"])
def test_device_pools_past_2_31_and_2_32(pool, bound):
    """pipeline_cases.offsets through brc_plan_device / brc_run_device / brc_fetch_device_results with its quality (or base) pool
    starting at 2^k - δ, k = 31 or 32, for two δ: the boundary inside a read of a staged K0 block and a staged K1 chunk (K1
    addresses staged bytes with the low 32 bits of the offsets), and inside a read too long for any stage (full 64-bit
    offsets).  The run at offset 0 and the oracle give the same raw accumulators.  brc_run_device takes the offsets as given:
    no padding records are needed.  One run holds at most about 4.3 GB."""
    import torch
    from bam_readcount_b200.engine import admitted
    case = pc.offsets()
    odump = cases.run_oracle(case, dict(), site_list=True).dump
    region = case["regions"][0]
    tid, _, _, sub = cases.region_reads(case, *region)
    assert len(admitted(sub, tid, 10_000_000)) == sub.n_reads
    dev = torch.device("cuda", 0)
    deltas = _deltas(sub, pool)
    need = bound + (1 << 28)
    free, _ = torch.cuda.mem_get_info(dev)
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")
    with cases.open_engine(case) as e:
        s = torch.cuda.Stream(device=dev)
        for what, lead in [("offset 0", 0)] + [(f"δ {k}", bound - d) for k, d in deltas.items()]:
            cb, keep = cases.device_batch(sub, dev, lead=(pool, lead))
            if lead:
                off = np.asarray((sub.qual_off if pool == "qual" else sub.seq_off), np.int64) + lead
                assert off[0] < bound < off[-1], what                  # the run's offsets do cross the boundary
            edump = cases.run_device(e, case, region, cb, s)
            assert edump == odump, f"{pool} pool, {what}: " + first_diff(edump, odump)
            del keep, cb
            torch.cuda.synchronize(dev)
            torch.cuda.empty_cache()
