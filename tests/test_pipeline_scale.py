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
import hashlib
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import cases
import pipeline_cases as pc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bam_readcount_b200", "csrc")
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _first_diff(a: str, b: str) -> str:
    la, lb = a.splitlines(), b.splitlines()
    for i, (x, y) in enumerate(zip(la, lb)):
        if x != y:
            return f"line {i}:\n got: {x[:300]}\nwant: {y[:300]}"
    return f"length differs: got {len(la)} lines, want {len(lb)}"


@functools.lru_cache(maxsize=None)
def _select_kernels() -> int:
    src = open(os.path.join(CSRC, "brc_device.cuh")).read()
    return int(re.search(r"constexpr\s+int\s+SELECT_KERNELS\s*=\s*(\d+);", src).group(1))


def _geometry(case, region):
    """(sub batch, first_pos, n_slots, n_tiles) of one region as brc_begin_region / brc_end_region form them."""
    tid, beg, end, sub = cases.region_reads(case, *region)
    first_pos = max(beg - 1, 0)
    n_slots = max(0, min(end, int(sub.ref_end().max())) - first_pos) if sub.n_reads else 0
    return sub, first_pos, n_slots, (n_slots + pc.TILE - 1) // pc.TILE


def _plan(case, n_chunks, region=None):
    sub, first_pos, n_slots, n_tiles = _geometry(case, region or case["regions"][0])
    return pc.pipe_plan(sub.pos, first_pos, n_tiles, n_chunks)


@functools.lru_cache(maxsize=None)
def _oracle(case_fn, fname, sl):
    return cases.run_oracle(case_fn(), cases.FLAG_SETS[fname], site_list=sl)


def _engine(case, flags, sl, filt=None):
    """One batch of the case's regions, each region's reads one push: (text, dump or "", warnings, launch count, pool records)."""
    from bam_readcount_b200.batch import ReadBatch
    from bam_readcount_b200.engine import Engine, admitted
    e = Engine(lib_names=case["lib_names"], **flags)
    try:
        name, clen, seq, wb = case["contigs"][0]
        e.set_reference(0, name, clen, seq, wb)
        if filt:
            e.set_site_filter(*filt)
        pushed = []
        for region in case["regions"]:
            tid, beg, end, sub = cases.region_reads(case, *region)
            e.begin_region(tid, beg, end, sl)
            e.push_reads(sub)
            e.end_region()
            pushed.append(sub.select(admitted(sub, tid, flags.get("max_cnt", 10_000_000))))
        res = e.compute()
        dump = res.dump(ReadBatch.concat(pushed), {0: (wb, seq)}) if res is not None else ""
        n_sec = e.packed().n_sec if res is not None else -1
        return e.format_text(-1), dump, e.warnings(), e.launch_count(), n_sec
    finally:
        e.close()


def _check(got, want, what):
    etext, edump, ewarn = got[:3]
    otext, odump, owarn = want
    assert edump == odump, f"{what}: " + _first_diff(edump, odump)
    assert etext == otext, f"{what}: " + _first_diff(etext, otext)
    assert (ewarn[0], ewarn[1], ewarn[3]) == owarn, what


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
def test_chunk_cuts_reach_every_edge_of_the_chunk_rule():
    for n_libs in (3, 12):
        case = pc.chunk_cuts(n_libs)
        sub, first_pos, n_slots, n_tiles = _geometry(case, case["regions"][0])
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
        sub, first_pos, n_slots, n_tiles = _geometry(carry, region)
        assert sub.n_reads < 2048 and sum(1 for _, _, t0, t1 in pc.pipe_plan(sub.pos, first_pos, n_tiles, 7) if t1 > t0) > 1


def test_deep_site_case_takes_the_deep_kernel():
    case = pc.deep_site()
    sub, first_pos, n_slots, n_tiles = _geometry(case, case["regions"][0])
    assert sub.n_reads >= 2048 and n_slots <= 2 and n_tiles == 1


JOBS = pc.jobs()


@pytest.mark.parametrize("job", JOBS, ids=[j[4] for j in JOBS])
def test_oracle_equals_reference_binary_on_pipeline_cases(job):
    with open(os.path.join(GOLDEN, "pipeline_sha256.json")) as fh:
        want = json.load(fh)
    case, fname, fl, sl, key = job
    got, _, _ = cases.run_oracle(case, fl, site_list=sl)
    assert hashlib.sha256(got.encode("latin-1")).hexdigest() == want[key], f"{key}: oracle differs from the reference binary"


# ---------------------------------------------------------------------------------------------------------------------------
# GPU: chunked push path
# ---------------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _one_chunk_text(fname):
    old = os.environ.get("BRC_PIPE_CHUNKS")
    os.environ["BRC_PIPE_CHUNKS"] = "1"
    try:
        return _engine(pc.chunk_cuts(3), cases.FLAG_SETS[fname], False)[0]
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
        want = _oracle(pc.chunk_cuts, fname, False)
        one = _one_chunk_text(fname)
        monkeypatch.setenv("BRC_PIPE_CHUNKS", str(n_chunks))
        got = _engine(case, fl, False)
        _check(got, want, f"{n_chunks} chunks, {fname}")
        assert got[0] == one, f"{n_chunks} chunks, {fname}: text differs from one chunk"
        assert got[3] == (3 if "max_cnt" in fl else pc.pipe_launches(plan)), (fname, got[3])
    if n_chunks > 1:                # word copies of later chunks start past slot 0; pool records leave in pieces
        assert any(t0 > 0 and t1 > t0 for _, _, t0, t1 in plan) and got[4] > 0


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
        want = cases.run_oracle(case, fl, site_list=False)
        got = _engine(case, fl, False)
        _check(got, want, f"{n_libs} libraries, {n_chunks} chunks, {fname}")
        assert got[3] == pc.pipe_launches(plan)


@pytest.mark.gpu
@pytest.mark.parametrize("n_chunks", [7, 65])
def test_multi_chunk_site_filter(n_chunks, monkeypatch):
    """With a site filter, the chunk loop skips the per-chunk copies and the selection kernels run after it: the filtered text is
    select_lines (tests/test_site_filter.py's restatement) of the oracle's."""
    from test_site_filter import THRESHOLDS, select_lines
    case = pc.chunk_cuts(3)
    plan = _plan(case, n_chunks)
    monkeypatch.setenv("BRC_PIPE_CHUNKS", str(n_chunks))
    for fname in ("default", "perlib"):
        otext = _oracle(pc.chunk_cuts, fname, False)[0]
        for mc, mf in THRESHOLDS:
            text, _, _, launches, _ = _engine(case, cases.FLAG_SETS[fname], False, filt=(mc, mf))
            want = select_lines(otext, mc, mf)
            assert text == want, (fname, mc, mf, _first_diff(text, want))
            assert launches == pc.pipe_launches(plan, selection_kernels=_select_kernels()), (fname, launches)


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [dict(), dict(per_lib=True)], ids=["alllib", "perlib"])
@pytest.mark.parametrize("n_chunks", [7, 65])
def test_multi_chunk_pool_overflow_falls_back(flags, n_chunks, monkeypatch):
    """test_kernel_boundaries.pool_case (random bases: four or five base classes per site) in many chunks: compute_pipelined's pool
    overflows, brc_compute falls back to the plain path, which grows the pool.  The fallback shows in the launch count (the plain
    path's three, not the chunk plan's) and in a pool larger than its initial capacity."""
    from test_kernel_boundaries import _initial_pool_cap, pool_case
    case = pool_case()
    plan = _plan(case, n_chunks)
    assert pc.pipe_launches(plan) > 3 + n_chunks
    monkeypatch.setenv("BRC_PIPE_CHUNKS", str(n_chunks))
    want = cases.run_oracle(case, flags, site_list=True)
    got = _engine(case, flags, True)
    _check(got, want, f"{n_chunks} chunks")
    assert got[3] == 3, f"launch count {got[3]}: the pipelined run did not fall back"
    _, _, n_slots, _ = _geometry(case, case["regions"][0])
    assert got[4] > _initial_pool_cap(case, flags, n_slots)


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
    want = cases.run_oracle(case, flags, site_list=True)
    got = _engine(case, flags, True)
    _check(got, want, f"{n_chunks} chunks")
    assert got[3] == pc.pipe_launches(plan, n_deep=1), got[3]


@pytest.mark.gpu
@pytest.mark.parametrize("fname", ["default", "perlib"])
def test_multi_chunk_carried_queue(fname, monkeypatch):
    """brc_set_queue_carry on: four adjacent and overlapping argv regions, one brc_compute each, each region's reads one borrowed
    push in 7 chunks.  The concatenated text equals the four regions as one batch, and the oracle's."""
    from bam_readcount_b200.engine import Engine
    case = pc.carried_regions()
    fl = cases.FLAG_SETS[fname]
    otext = _oracle(pc.carried_regions, fname, False)[0]
    one = _engine(case, fl, False)[0]
    assert one == otext, _first_diff(one, otext)
    monkeypatch.setenv("BRC_PIPE_CHUNKS", "7")
    e = Engine(lib_names=case["lib_names"], **fl)
    try:
        name, clen, seq, wb = case["contigs"][0]
        e.set_reference(0, name, clen, seq, wb)
        assert e.lib.brc_set_queue_carry(e.h, 1) == 0
        parts = []
        for region in case["regions"]:
            tid, beg, end, sub = cases.region_reads(case, *region)
            e.reset()
            e.begin_region(tid, beg, end, False)
            e.push_reads(sub)
            e.end_region()
            e.compute()
            assert e.launch_count() == pc.pipe_launches(_plan(case, 7, region)), region
            parts.append(e.format_text(-1))
        assert "".join(parts) == one, _first_diff("".join(parts), one)
    finally:
        e.close()


# ---------------------------------------------------------------------------------------------------------------------------
# GPU: one CTA per SM
# ---------------------------------------------------------------------------------------------------------------------------
def _starved_jobs():
    from test_kernel_boundaries import pool_case, selection_cases
    import boundary_cases
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
        otext, odump, owarn = cases.run_oracle(case, flags, site_list=sl)
        if n_chunks:
            os.environ["BRC_PIPE_CHUNKS"] = str(n_chunks)
            try:
                etext, edump, ewarn, launches, _ = _engine(case, flags, sl)
            finally:
                del os.environ["BRC_PIPE_CHUNKS"]
        else:
            (etext, edump, ewarn, _), launches = cases.run_engine(case, flags, site_list=sl), 0
        out[name] = dict(dump=edump == odump, text=etext == otext, warn=[ewarn[0], ewarn[1], ewarn[3]] == list(owarn),
                         launches=launches, diff="" if edump == odump else _first_diff(edump, odump))
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
    _, _, _, n_tiles = _geometry(big, big["regions"][0])
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
    from test_kernel_boundaries import k1_chunks, kernel_constants, tile_ranges
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
    sub, first_pos, n_slots, _ = _geometry(case, case["regions"][0])
    for pool in ("qual", "seq"):
        for bound in (1 << 31, 1 << 32):
            d = _deltas(sub, pool)
            assert _straddles(sub, pool, bound - d["staged"], bound, first_pos, n_slots)[:2] == (True, True), (pool, bound)
            assert _straddles(sub, pool, bound - d["long"], bound, first_pos, n_slots)[2], (pool, bound)


def _device_batch_at(b, pool, lead, device):
    """The batch's arrays on the device, the quality (or base) pool placed `lead` bytes into an allocation whose first `lead` bytes
    are never written, its offsets shifted by `lead`."""
    import torch
    from bam_readcount_b200.engine import CReadBatch
    view = {np.dtype(np.uint16): np.int16, np.dtype(np.uint32): np.int32, np.dtype(np.uint64): np.int64}
    keep = []

    def dev(a, pad=0, lead_=0):
        a = np.ascontiguousarray(a)
        a = a.view(view.get(a.dtype, a.dtype))
        if lead_:
            t = torch.empty(lead_ + a.shape[0] + pad, dtype=torch.uint8, device=device)
            t[lead_:lead_ + a.shape[0]].copy_(torch.from_numpy(a))
            t[lead_ + a.shape[0]:].zero_()
        else:
            t = torch.from_numpy(np.concatenate([a, np.zeros(pad, a.dtype)]) if pad else a).to(device)
        keep.append(t)
        return t.data_ptr()
    shift = lambda off, p: (off.astype(np.uint64) + np.uint64(lead if pool == p else 0))
    ptrs = [dev(b.tid), dev(b.pos), dev(b.flag), dev(b.mapq), dev(b.lib), dev(b.l_qseq), dev(b.nm), dev(b.sm), dev(b.cigar_off),
            dev(b.cigar), dev(shift(b.seq_off, "seq")), dev(b.seq, 64, lead if pool == "seq" else 0),
            dev(shift(b.qual_off, "qual")), dev(b.qual, 64, lead if pool == "qual" else 0)]
    return CReadBatch(b.n_reads, *ptrs), keep


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
    from bam_readcount_b200.engine import CRegion, Engine, admitted
    case = pc.offsets()
    _, odump, _ = cases.run_oracle(case, dict(), site_list=True)
    region = case["regions"][0]
    tid, beg, end, sub = cases.region_reads(case, *region)
    _, first_pos, n_slots, _ = _geometry(case, region)
    assert len(admitted(sub, tid, 10_000_000)) == sub.n_reads
    dev = torch.device("cuda", 0)
    deltas = _deltas(sub, pool)
    need = bound + (1 << 28)
    free, _ = torch.cuda.mem_get_info(dev)
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")
    name, clen, seq, wb = case["contigs"][0]
    e = Engine(lib_names=case["lib_names"])
    try:
        e.set_reference(tid, name, clen, seq, wb)
        s = torch.cuda.Stream(device=dev)
        e.plan_device([CRegion(tid, beg, end, 1, 0, sub.n_reads, 0, first_pos, n_slots)], sub.n_reads, 1 << 20)
        for what, lead in [("offset 0", 0)] + [(f"δ {k}", bound - d) for k, d in deltas.items()]:
            cb, keep = _device_batch_at(sub, pool, lead, dev)
            if lead:
                off = np.asarray((sub.qual_off if pool == "qual" else sub.seq_off), np.int64) + lead
                assert off[0] < bound < off[-1], what                  # the run's offsets do cross the boundary
            e.run_device(cb, None, s.cuda_stream)
            res = e.fetch_device_results(s.cuda_stream)
            edump = res.dump(sub, {tid: (wb, seq)})
            assert edump == odump, f"{pool} pool, {what}: " + _first_diff(edump, odump)
            del keep, cb
            torch.cuda.synchronize(dev)
            torch.cuda.empty_cache()
    finally:
        e.close()
