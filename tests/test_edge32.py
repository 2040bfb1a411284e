"""The kernels at their 32-bit edges (tests/edge32_cases.py), bit for bit against the oracle.

CPU
  audit    for every boundary and target the CIGAR-offset runs reach what they claim: a staged-CIGAR K1 chunk whose op window
           straddles the boundary with non-simple reads on both sides, an unstaged chunk whose non-simple reads start at or past
           it, deep-site tiles (by read count and forced) and an indel look-ahead whose ops lie past it.  The 2^31 cases admit
           reads ending past INT32_MAX that cover printed sites, and a warp window of their last tile reaches past INT32_MAX.
  anchor   the oracle's text on the 2^31 cases against the SHA-256 of what the unmodified reference binary printed
           (tests/golden/edge32_sha256.json, written by tests/golden/make_golden.py --edge32-only from a BAM indexed as CSI, since
           BAI cannot address past 2^29, and the whole 2 GiB FASTA: mostly N, the window's bases at its end).
GPU, each asserting that it reached its path
  test_device_cigar_pool_past_2_31_and_2_32   brc_run_device with the CIGAR pool at 2^k - δ ops, one δ per target, against the
                                              offset-0 run and the oracle; the lead-in holds 1M ops, so a kernel that resolves
                                              another read's ops reads short in-bounds CIGARs and fails as a mismatch.
  test_reads_past_2_31                        brc_push_reads and brc_run_device, deep-site kernel forced and not, against the
                                              oracle: raw accumulators, text and warning counters."""
import functools

import numpy as np
import pytest

import cases
import edge32_cases as ec
from cases import first_diff, region_geometry
from kernel_model import k1_chunks, tile_ranges

BOUNDS = (1 << 31, 1 << 32)


def _shifted(sub, lead):
    import dataclasses
    return dataclasses.replace(sub, cigar_off=sub.cigar_off.astype(np.uint64) + np.uint64(lead))


@functools.lru_cache(maxsize=None)
def _targets():
    """target -> (region, site_list, δ, site)"""
    case = ec.cigar_offsets()
    out = {}
    for target, (ri, sl) in ec.CIGAR_TARGETS.items():
        region = case["regions"][ri]
        _, _, _, sub, first_pos, n_slots, _ = region_geometry(case, region)
        chunks = k1_chunks(sub, tile_ranges(sub, first_pos, first_pos + n_slots))
        site = region[1] - 1
        out[target] = (ri, sl, ec.cigar_target_delta(sub, target, chunks, site), site)
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bound", BOUNDS, ids=["2^31", "2^32"])
def test_cigar_offset_runs_reach_their_targets(bound):
    case = ec.cigar_offsets()
    for target, (ri, sl, delta, site) in _targets().items():
        _, _, _, sub, first_pos, n_slots, _ = region_geometry(case, case["regions"][ri])
        lead = bound - delta
        b = _shifted(sub, lead)
        co = b.cigar_off.astype(np.int64)
        ns = ec._nonsimple(b)
        assert co[0] < bound <= co[-1], target                          # the run's op offsets cross the boundary
        if target in ("staged", "unstaged"):
            chunks = k1_chunks(b, tile_ranges(sub, first_pos, first_pos + n_slots))   # tiles do not depend on the offsets
            if target == "staged":
                hit = [c for c in chunks if c["cstaged"] and (co[c["r0"]] & ~3) < bound < ((co[c["r1"]] + 3) & ~3)
                       and any(ns[i] and co[i] < bound for i in range(c["r0"], c["r1"]))
                       and any(ns[i] and co[i] >= bound for i in range(c["r0"], c["r1"]))]
            else:
                hit = [c for c in chunks if not c["cstaged"] and any(ns[i] for i in range(c["r0"], c["r1"]))
                       and all(co[i] >= bound for i in range(c["r0"], c["r1"]) if ns[i])]
            assert hit, (target, bound)
        else:
            # a site-list line: one tile of one site; its reads (all of them cover it) past the boundary include non-simple ones
            # >= 2048 reads (the engine's deep_min_reads) takes the deep-site kernel unforced
            assert n_slots <= 2 and (sub.n_reads >= 2048) == (target in ("deep", "lookahead")), (target, sub.n_reads)
            past = [i for i in range(sub.n_reads) if co[i] >= bound and ns[i]]
            assert len(past) > 50, target
            if target == "lookahead":
                assert ec.indel_at(sub, int(np.searchsorted(co, bound)), site) != 0   # the first read past it ends an M op there


def test_reads_past_2_31_cover_printed_sites():
    from bam_readcount_b200.engine import admitted
    for k in ec.END_KS:
        case = ec.contig_end_2_31(k)
        L = case["contigs"][0][1]
        assert L == 2 ** 31 - 1 - k and case["contigs"][0][3] > 0
        tid, beg, end, sub, first_pos, n_slots, _ = region_geometry(case, case["regions"][0])
        assert end == L and n_slots % 256 == 2 and first_pos + n_slots == L      # the last tile holds the last two sites
        e = sub.ref_end()
        adm = admitted(sub, tid, 10_000_000)
        past = [i for i in adm if int(e[i]) > ec.INT32_MAX]
        assert past, k
        assert {int(sub.flag[i]) & 16 for i in past} == {0, 16}                # both strands
        assert all(int(sub.pos[i]) <= L - 3 < L - 1 < int(e[i]) for i in past[:20])   # they cover the last sites
        if k < 30:
            assert first_pos + n_slots - 2 + 31 >= ec.INT32_MAX            # the last tile's warp window reaches past INT32_MAX


EDGE_JOBS = ec.jobs()


@pytest.mark.parametrize("job", EDGE_JOBS, ids=[j[4] for j in EDGE_JOBS])
def test_oracle_equals_reference_binary_on_reads_past_2_31(job):
    case, fname, fl, sl, key = job
    cases.assert_anchor("edge32_sha256.json", key, cases.run_oracle(case, fl, site_list=sl).text)


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("bound", BOUNDS, ids=["2^31", "2^32"])
def test_device_cigar_pool_past_2_31_and_2_32(bound, monkeypatch):
    """cigar_offsets through brc_plan_device / brc_run_device / brc_fetch_device_results, one region per plan, with the CIGAR pool
    starting at 2^k - δ ops of an allocation whose lead-in holds 1M ops: per target, the boundary inside a staged-CIGAR K1 chunk
    (ops addressed in shared memory relative to the chunk's first op), before the non-simple reads of an unstaged chunk (global
    loads), under a deep-site tile by read count and one forced, and before an indel anchored at the deep site (the look-ahead
    at the next op).  Each run's raw accumulators equal the offset-0 run's and the oracle's.  One run holds about 16.3 GiB."""
    import torch
    from bam_readcount_b200.engine import admitted
    dev = torch.device("cuda", 0)
    case = ec.cigar_offsets()
    targets = _targets()
    n_ops_max = max(int(cases.region_reads(case, *r)[3].cigar.shape[0]) for r in case["regions"])
    need = 4 * (bound + n_ops_max) + (1 << 30)
    free, _ = torch.cuda.mem_get_info(dev)
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")
    pool = torch.full((bound + n_ops_max + 16,), 0x10, dtype=torch.int32, device=dev)       # 1M ops
    s = torch.cuda.Stream(device=dev)
    try:
        for target, (ri, sl, delta, site) in targets.items():
            region = case["regions"][ri]
            tid, _, _, sub = cases.region_reads(case, *region)
            assert len(admitted(sub, tid, 10_000_000)) == sub.n_reads
            odump = cases.run_oracle(dict(case, regions=[region]), dict(), site_list=sl).dump
            if target == "deep_forced":
                monkeypatch.setenv("BRC_DEEP_MIN_READS", "1")
            else:
                monkeypatch.delenv("BRC_DEEP_MIN_READS", raising=False)
            with cases.open_engine(case) as e:
                cb, keep = cases.device_batch(sub, dev)
                d0 = cases.run_device(e, case, region, cb, s, site_list=sl)
                assert d0 == odump, f"{target}, offset 0: " + first_diff(d0, odump)
                if target in ("deep", "deep_forced", "lookahead"):
                    assert e.launch_count() == 4, (target, e.launch_count())  # init, K0, pileup, deep-site kernel
                lead = bound - delta
                n = sub.cigar.shape[0]
                cb, keep = cases.device_batch(sub, dev, cigar_pool=(pool, lead))
                assert int(sub.cigar_off[0]) + lead < bound <= int(sub.cigar_off[-1]) + lead, target
                dl = cases.run_device(e, case, region, cb, s, site_list=sl)
                pool[lead:lead + n].fill_(0x10)
                assert dl == odump, f"{target}, δ {delta} before 2^{bound.bit_length() - 1}: " + first_diff(dl, odump)
                del cb, keep
    finally:
        del pool
        torch.cuda.synchronize(dev)
        torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("k", ec.END_KS)
def test_reads_past_2_31(k, monkeypatch):
    """contig_end_2_31(k): the argv region to the contig end and the site-list lines of its last three positions, with the flag
    sets default, -p and -i, through brc_push_reads (raw accumulators, text, warning counters) and, for the argv region,
    brc_run_device (raw accumulators); each with the deep-site kernel forced (BRC_DEEP_MIN_READS=1: the argv region's last tile of
    two sites and every site-list line go to it) and not (both go to pileup_kernel)."""
    import torch
    case = ec.contig_end_2_31(k)
    lines = ec.site_lines(case)
    dev = torch.device("cuda", 0)
    s = torch.cuda.Stream(device=dev)
    for forced in (False, True):
        if forced:
            monkeypatch.setenv("BRC_DEEP_MIN_READS", "1")
        else:
            monkeypatch.delenv("BRC_DEEP_MIN_READS", raising=False)
        for fname in ec.END_FLAGS:
            fl = cases.FLAG_SETS[fname]
            for c, sl in ((case, False), (lines, True)):
                want = cases.run_oracle(c, fl, site_list=sl)
                assert len(want.text.splitlines()) >= (3 if sl else 19000)
                what = f"k={k}, {fname}, {'site list' if sl else 'argv'}, deep {'forced' if forced else 'auto'}"
                cases.assert_same(cases.run_engine(c, fl, site_list=sl), want, what)
            # the device path: the argv region's reads resident on the device
            region = case["regions"][0]
            odump = cases.run_oracle(case, fl, site_list=False).dump
            with cases.open_engine(case, fl) as e:
                cb, keep = cases.device_batch(cases.region_reads(case, *region)[3], dev)
                edump = cases.run_device(e, case, region, cb, s, site_list=False)
                assert edump == odump, f"k={k}, {fname}, device path, deep {'forced' if forced else 'auto'}: " + first_diff(edump, odump)
                # the last tile (two sites) is a deep-site candidate: the region holds more than 2048 reads; its own ~150 reads go
                # to deep_site_kernel only when forced, and to pileup_kernel otherwise
                assert e.launch_count() == 4, e.launch_count()
