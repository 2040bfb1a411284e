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
import hashlib
import json
import os

import numpy as np
import pytest

import cases
import edge32_cases as ec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
BOUNDS = (1 << 31, 1 << 32)


def _first_diff(a: str, b: str) -> str:
    la, lb = a.splitlines(), b.splitlines()
    for i, (x, y) in enumerate(zip(la, lb)):
        if x != y:
            return f"line {i}:\n got: {x[:300]}\nwant: {y[:300]}"
    return f"length differs: got {len(la)} lines, want {len(lb)}"


def _geometry(case, region):
    """(tid, beg, end, sub batch, first_pos, n_slots) of one region as brc_begin_region / brc_end_region form them."""
    tid, beg, end, sub = cases.region_reads(case, *region)
    first_pos = max(beg - 1, 0)
    n_slots = max(0, min(end, int(sub.ref_end().max())) - first_pos) if sub.n_reads else 0
    return tid, beg, end, sub, first_pos, n_slots


def _shifted(sub, lead):
    import dataclasses
    return dataclasses.replace(sub, cigar_off=sub.cigar_off.astype(np.uint64) + np.uint64(lead))


@functools.lru_cache(maxsize=None)
def _targets():
    """target -> (region, site_list, δ, site)"""
    from test_kernel_boundaries import k1_chunks, tile_ranges
    case = ec.cigar_offsets()
    out = {}
    for target, (ri, sl) in ec.CIGAR_TARGETS.items():
        region = case["regions"][ri]
        _, _, _, sub, first_pos, n_slots = _geometry(case, region)
        chunks = k1_chunks(sub, tile_ranges(sub, first_pos, first_pos + n_slots))
        site = region[1] - 1
        out[target] = (ri, sl, ec.cigar_target_delta(sub, target, chunks, site), site)
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bound", BOUNDS, ids=["2^31", "2^32"])
def test_cigar_offset_runs_reach_their_targets(bound):
    from test_kernel_boundaries import k1_chunks, tile_ranges
    case = ec.cigar_offsets()
    for target, (ri, sl, delta, site) in _targets().items():
        _, _, _, sub, first_pos, n_slots = _geometry(case, case["regions"][ri])
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
        tid, beg, end, sub, first_pos, n_slots = _geometry(case, case["regions"][0])
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
    with open(os.path.join(GOLDEN, "edge32_sha256.json")) as fh:
        want = json.load(fh)
    case, fname, fl, sl, key = job
    got, _, _ = cases.run_oracle(case, fl, site_list=sl)
    assert hashlib.sha256(got.encode("latin-1")).hexdigest() == want[key], f"{key}: oracle differs from the reference binary"


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
def _device_arrays(b, device):
    """Every array of the batch but the CIGAR pool and its offsets on the device (64 spare bytes behind the byte pools)."""
    import torch
    view = {np.dtype(np.uint16): np.int16, np.dtype(np.uint32): np.int32, np.dtype(np.uint64): np.int64}

    def dev(a, pad=0):
        a = np.ascontiguousarray(a)
        a = a.view(view.get(a.dtype, a.dtype))
        if pad:
            a = np.concatenate([a, np.zeros(pad, a.dtype)])
        return torch.from_numpy(a).to(device)
    return dict(tid=dev(b.tid), pos=dev(b.pos), flag=dev(b.flag), mapq=dev(b.mapq), lib=dev(b.lib), l_qseq=dev(b.l_qseq), nm=dev(b.nm),
                sm=dev(b.sm), seq_off=dev(b.seq_off), seq=dev(b.seq, 64), qual_off=dev(b.qual_off), qual=dev(b.qual, 64))


def _cbatch(t, n, cigar_off, cigar_ptr):
    from bam_readcount_b200.engine import CReadBatch
    return CReadBatch(n, t["tid"].data_ptr(), t["pos"].data_ptr(), t["flag"].data_ptr(), t["mapq"].data_ptr(), t["lib"].data_ptr(),
                      t["l_qseq"].data_ptr(), t["nm"].data_ptr(), t["sm"].data_ptr(), cigar_off.data_ptr(), cigar_ptr,
                      t["seq_off"].data_ptr(), t["seq"].data_ptr(), t["qual_off"].data_ptr(), t["qual"].data_ptr())


def _device_dump(e, sub, t, cigar_off, cigar_ptr, stream, tid, wb, seq):
    e.run_device(_cbatch(t, sub.n_reads, cigar_off, cigar_ptr), None, stream.cuda_stream)
    return e.fetch_device_results(stream.cuda_stream).dump(sub, {tid: (wb, seq)})


@pytest.mark.gpu
@pytest.mark.parametrize("bound", BOUNDS, ids=["2^31", "2^32"])
def test_device_cigar_pool_past_2_31_and_2_32(bound, monkeypatch):
    """cigar_offsets through brc_plan_device / brc_run_device / brc_fetch_device_results, one region per plan, with the CIGAR pool
    starting at 2^k - δ ops of an allocation whose lead-in holds 1M ops: per target, the boundary inside a staged-CIGAR K1 chunk
    (ops addressed in shared memory relative to the chunk's first op), before the non-simple reads of an unstaged chunk (global
    loads), under a deep-site tile by read count and one forced, and before an indel anchored at the deep site (the look-ahead
    at the next op).  Each run's raw accumulators equal the offset-0 run's and the oracle's.  One run holds about 16.3 GiB."""
    import torch
    from bam_readcount_b200.engine import CRegion, Engine, admitted
    dev = torch.device("cuda", 0)
    case = ec.cigar_offsets()
    targets = _targets()
    n_ops_max = max(int(cases.region_reads(case, *r)[3].cigar.shape[0]) for r in case["regions"])
    need = 4 * (bound + n_ops_max) + (1 << 30)
    free, _ = torch.cuda.mem_get_info(dev)
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")
    pool = torch.full((bound + n_ops_max + 16,), 0x10, dtype=torch.int32, device=dev)       # 1M ops
    name, clen, seq, wb = case["contigs"][0]
    s = torch.cuda.Stream(device=dev)
    try:
        for target, (ri, sl, delta, site) in targets.items():
            region = case["regions"][ri]
            tid, beg, end, sub, first_pos, n_slots = _geometry(case, region)
            assert len(admitted(sub, tid, 10_000_000)) == sub.n_reads
            _, odump, _ = cases.run_oracle(dict(case, regions=[region]), dict(), site_list=sl)
            if target == "deep_forced":
                monkeypatch.setenv("BRC_DEEP_MIN_READS", "1")
            else:
                monkeypatch.delenv("BRC_DEEP_MIN_READS", raising=False)
            e = Engine(lib_names=case["lib_names"])
            try:
                e.set_reference(tid, name, clen, seq, wb)
                e.plan_device([CRegion(tid, beg, end, 1 if sl else 0, 0, sub.n_reads, 0, first_pos, n_slots)], sub.n_reads, 1 << 20)
                t = _device_arrays(sub, dev)
                cig = torch.from_numpy(sub.cigar.view(np.int32)).to(dev)
                off0 = torch.from_numpy(sub.cigar_off.view(np.int64)).to(dev)
                d0 = _device_dump(e, sub, t, off0, cig.data_ptr(), s, tid, wb, seq)
                assert d0 == odump, f"{target}, offset 0: " + _first_diff(d0, odump)
                if target in ("deep", "deep_forced", "lookahead"):
                    assert e.launch_count() == 4, (target, e.launch_count())  # init, K0, pileup, deep-site kernel
                lead = bound - delta
                n = sub.cigar.shape[0]
                pool[lead:lead + n].copy_(cig)
                offl = torch.from_numpy((sub.cigar_off.astype(np.uint64) + np.uint64(lead)).view(np.int64)).to(dev)
                assert int(offl[0]) < bound <= int(offl[-1]), target
                dl = _device_dump(e, sub, t, offl, pool.data_ptr(), s, tid, wb, seq)
                pool[lead:lead + n].fill_(0x10)
                assert dl == odump, f"{target}, δ {delta} before 2^{bound.bit_length() - 1}: " + _first_diff(dl, odump)
                del t, cig, off0, offl
            finally:
                e.close()
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
    from bam_readcount_b200.engine import CRegion, Engine
    case = ec.contig_end_2_31(k)
    lines = ec.site_lines(case)
    name, clen, seq, wb = case["contigs"][0]
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
                otext, odump, owarn = cases.run_oracle(c, fl, site_list=sl)
                assert len(otext.splitlines()) >= (3 if sl else 19000)
                etext, edump, ewarn, _ = cases.run_engine(c, fl, site_list=sl)
                what = f"k={k}, {fname}, {'site list' if sl else 'argv'}, deep {'forced' if forced else 'auto'}"
                assert edump == odump, what + ": " + _first_diff(edump, odump)
                assert etext == otext, what + ": " + _first_diff(etext, otext)
                assert (ewarn[0], ewarn[1], ewarn[3]) == owarn, what
            # the device path: the argv region's reads resident on the device
            tid, beg, end, sub, first_pos, n_slots = _geometry(case, case["regions"][0])
            _, odump, _ = cases.run_oracle(case, fl, site_list=False)
            e = Engine(lib_names=case["lib_names"], **fl)
            try:
                e.set_reference(tid, name, clen, seq, wb)
                e.plan_device([CRegion(tid, beg, end, 0, 0, sub.n_reads, 0, first_pos, n_slots)], sub.n_reads, 1 << 20)
                t = _device_arrays(sub, dev)
                cig = torch.from_numpy(sub.cigar.view(np.int32)).to(dev)
                off = torch.from_numpy(sub.cigar_off.view(np.int64)).to(dev)
                edump = _device_dump(e, sub, t, off, cig.data_ptr(), s, tid, wb, seq)
                assert edump == odump, f"k={k}, {fname}, device path, deep {'forced' if forced else 'auto'}: " + _first_diff(edump, odump)
                # the last tile (two sites) is a deep-site candidate: the region holds more than 2048 reads; its own ~150 reads go
                # to deep_site_kernel only when forced, and to pileup_kernel otherwise
                assert e.launch_count() == 4, e.launch_count()
            finally:
                e.close()
