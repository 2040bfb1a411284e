"""The kernels at their capacity limits (tests/boundary_cases.py), bit for bit.

CPU
  audit   the capacities are parsed out of csrc/; from each case's batch the test recomputes what the kernels will decide (K0's
          staged blocks and reference window, the producer's chunk cuts and CIGAR staging, FM_FASTDIV / FM_HOT per read, per-site
          depth and 16-bit sums, deep-tile read counts) and asserts that every target of the case lands on both sides of its
          limit.  If a constant changes, the failing target names the case that no longer straddles it.
  anchor  the oracle's text on every case and flag set against the SHA-256 of what the unmodified reference binary printed
          (tests/golden/boundary_sha256.json, written by tests/golden/make_golden.py).
GPU
  the engine against the oracle on every case and flag set (raw accumulators, text, warning counters), forced through the
  deep-site kernel, as one borrowed push and as two pushes; the reciprocal-division self-test over every hot-path numerator;
  secondary-pool growth; the site selection at scale."""
import os
import re

import numpy as np
import pytest

import boundary_cases
import cases
from boundary_cases import initial_pool_cap, pool_case, selection_cases
from cases import first_diff
from kernel_model import (CONST_NAMES, CSRC, FM_FASTDIV, FM_HOT, FM_SIMPLE, cigar_shape, k0_blocks, k0_descriptors, k1_chunks,
                          kernel_constants, tile_ranges)
from site_filter_rule import THRESHOLDS, select_lines


# ---------------------------------------------------------------------------------------------------------------------------
# what the kernels decide, recomputed on the host (beyond kernel_model's)
# ---------------------------------------------------------------------------------------------------------------------------
def _reads_view(b):
    """Per read: list of (len, op char) and the decoded quality / base arrays."""
    ops = "MIDNSHP=XB"
    co = b.cigar_off.astype(np.int64)
    out = []
    for i in range(b.n_reads):
        out.append([(int(c) >> 4, ops[int(c) & 15]) for c in b.cigar[co[i]:co[i + 1]]])
    return out


def read_model(case, batch, site_list):
    """Per read, the descriptor K0 writes for it (kernel_model.k0_descriptors, the model tests/test_k0_descriptors.py holds the
    device to) as the targets below read it, with its CIGAR as (len, op char) pairs and its qoff."""
    contig = case["contigs"][0]
    region = dict(ref=0, site_list=site_list, first_pos=0, n_slots=0, read_lo=0, read_hi=batch.n_reads)
    d, _, _ = k0_descriptors(batch, [region], [contig], {})
    _, qoff = cigar_shape(batch)
    return [dict(lq=int(batch.l_qseq[i]), clen=int(d["clen"][i]), lclip=int(d["lclip"][i]), fast=bool(d["fm"][i] & FM_FASTDIV),
                 hot=bool(d["fm"][i] & FM_HOT), simple=bool(d["fm"][i] & FM_SIMPLE), qoff=int(qoff[i]), mmq=int(d["mmq"][i]),
                 se=int(d["se"][i]), ops=ops) for i, ops in enumerate(_reads_view(batch))]


def site_sums(batch, facts, lo, hi):
    """Per site in [lo, hi): depth, and the clipped-length / SE / mismatch-quality sums over covering live reads (every event of
    the stacks that target the 16-bit sums passes and lands in the primary class)."""
    n = hi - lo
    depth = np.zeros(n + 1, np.int64); clip = np.zeros(n + 1, np.int64); se = np.zeros(n + 1, np.int64); mmq = np.zeros(n + 1, np.int64)
    e = batch.ref_end()
    for i, f in enumerate(facts):
        a, b = max(int(batch.pos[i]), lo) - lo, min(int(e[i]), hi) - lo
        if b <= a:
            continue
        depth[a] += 1; depth[b] -= 1
        if batch.flag[i] & 1024:
            continue
        clip[a] += f["clen"]; clip[b] -= f["clen"]
        se[a] += f["se"] & 0xFFFFFFFF; se[b] -= f["se"] & 0xFFFFFFFF
        mmq[a] += f["mmq"]; mmq[b] -= f["mmq"]
    return {k: np.cumsum(v)[:n] for k, v in (("depth", depth), ("clip", clip), ("se", se), ("mmq", mmq))}


def _both(lo_side, hi_side, what):
    assert lo_side and hi_side, f"{what}: below the limit {'hit' if lo_side else 'MISSED'}, above it {'hit' if hi_side else 'MISSED'}"


def check_targets(case):
    K = kernel_constants()
    T = K["TILE"]
    ci, b1, e1 = case["regions"][0]
    tid, beg, end, batch = cases.region_reads(case, ci, b1, e1)
    if batch.n_reads != case["batch"].n_reads:      # site-list cases: per-read facts over every read of the case
        batch = case["batch"]
    facts = read_model(case, batch, case["site_list"])
    first_pos = max(beg, 0)
    for target in case["targets"]:
        if target == "k0_qual_cap":
            bl = [b for b in k0_blocks(batch, case) if b["uniform"]]
            _both(any(b["staged"] and b["lq"] * K["K0_READS"] + 32 > K["K0_QUAL_CAP"] - 160 for b in bl),
                  any(not b["staged"] and b["lq"] * K["K0_READS"] <= K["K0_QUAL_CAP"] + 160 for b in bl), target)
        elif target == "k1_stage_shrink":
            ch = [c for c in k1_chunks(batch, tile_ranges(batch, first_pos, end)) if c["full"] == K["STAGE_READS"] and len(c["lq"]) == 1]
            _both(any(c["r1"] - c["r0"] == c["full"] and c["staged"] and max(c["lq"]) * K["STAGE_READS"] + 32 == K["STAGE_QUAL"] for c in ch),
                  any(c["r1"] - c["r0"] < c["full"] and c["staged"] and max(c["lq"]) * K["STAGE_READS"] + 32 == K["STAGE_QUAL"] + K["STAGE_READS"]
                      for c in ch), target)
        elif target == "fastdiv_len":
            M = K["FASTDIV_MAX"]
            _both(any(f["lq"] == M and f["fast"] for f in facts), any(f["lq"] == M + 1 and not f["fast"] for f in facts), target)
        elif target == "fastdiv_clen":
            M = K["FASTDIV_MAX"]
            _both(any(f["clen"] == M and f["lq"] > M and not f["fast"] for f in facts) and any(f["clen"] == M and f["fast"] for f in facts),
                  any(f["clen"] == M + 1 and not f["fast"] for f in facts), target)
        elif target == "fastdiv_numerator":
            # largest |2 (qpos - left_clip) - clipped_length| of a hot read against the bound 2 b + 2 the self-test once stopped at:
            # the controls (soft clip first, or clips only at the end) stay inside it; nH mS kM reads on both strands go far past it
            def num(f):
                return max(abs(2 * (f["qoff"] - f["lclip"]) - f["clen"]), abs(2 * (f["qoff"] + f["clen"] - 1 - f["lclip"]) - f["clen"]))
            hot = [(i, f) for i, f in enumerate(facts) if f["hot"]]
            ctrl = [f for _, f in hot if f["ops"][0][1] != "H"]
            hs = [(i, f) for i, f in hot if f["ops"][0][1] == "H" and f["qoff"] > 0]
            _both(any(f["ops"][0][1] == "S" for f in ctrl) and any(f["ops"][0][1] == "M" for f in ctrl)
                  and all(num(f) <= 2 * f["clen"] + 2 for f in ctrl),
                  {int(batch.flag[i]) & 16 for i, _ in hs} == {0, 16} and all(num(f) > 2 * f["clen"] + 2 for _, f in hs)
                  and max(num(f) for _, f in hs) > 2 * K["FASTDIV_MAX"] - 100, target)
        elif target == "k0_ref_window":
            bl = k0_blocks(batch, case)
            _both(any(b["staged"] and b["ref_staged"] for b in bl),
                  any(b["ref_staged"] and b["past"] for b in bl) and any(b["staged"] and not b["ref_staged"] and b["span"] > 2 * K["K0_REF_CAP"]
                                                                          for b in bl), target)
        elif target == "chunk_reads":
            sizes = [h - l for l, h in tile_ranges(batch, first_pos, end)]
            S = K["STAGE_READS"]
            _both(S in sizes, S + 1 in sizes and 2 * S in sizes, target)
        elif target == "hot_run_end":
            ch = k1_chunks(batch, tile_ranges(batch, first_pos, end))
            full = [c for c in ch if c["r1"] - c["r0"] == K["STAGE_READS"]]

            def run_len(c):
                n = 0
                for i in range(c["r1"] - 1, c["r0"] - 1, -1):
                    if not facts[i]["hot"]:
                        break
                    n += 1
                return n
            _both(any(run_len(c) % 2 == 1 for c in full), any(run_len(c) % 2 == 0 and run_len(c) > 0 for c in full), target)
        elif target == "warp_edges":
            # in the tile built for it: reads starting at wfirst+31 / wfirst+32 and ending at wfirst / wfirst+1 of each probed warp
            pr = case["probe"]
            starts, ends = set(batch.pos.tolist()), set(batch.ref_end().tolist())
            wfs = [first_pos + pr["warp_tile"] * T + 32 * w for w in pr["warp_windows"]]
            _both(all(wf + 31 in starts and wf in ends for wf in wfs), all(wf + 32 in starts and wf + 1 in ends for wf in wfs), target)
        elif target == "tile_edges":
            starts = set(batch.pos.tolist())
            t0s = [first_pos + t * T for t in case["probe"]["edge_tiles"]]
            _both(all(t0 - 1 in starts for t0 in t0s), all(t0 in starts for t0 in t0s), target)
        elif target == "lead_skip":
            # the tile built for it: more than one ballot (32) of leading reads that end before its last warp's window, then reads
            # that cover that window
            t = case["probe"]["lead_tile"]
            l, h = tile_ranges(batch, first_pos, end)[t]
            last_w = first_pos + t * T + T - 32
            e_ = batch.ref_end()
            lead = 0
            while l + lead < h and e_[l + lead] <= last_w:
                lead += 1
            _both(any(e_[i] > last_w for i in range(l + lead, h)), lead > 32, target)
        elif target == "libless_hot":
            # the tile built for it: hot pairs of reads with a library (the pair body under -p), and a library-less read between two
            # such hot reads (never part of a pair)
            l, h = tile_ranges(batch, first_pos, end)[case["probe"]["libless_tile"]]
            has = lambda i: facts[i]["hot"] and batch.lib[i] != 0xFFFF
            _both(any(has(i) and has(i + 1) for i in range(l, h - 1)),
                  any(batch.lib[i] == 0xFFFF and has(i - 1) and has(i + 1) for i in range(l + 1, h - 1)), target)
        elif target == "queue_rows":
            # an argv region's last site whose covering reads all sit in library rows >= SEL_LAST_ROWS, with a deletion anchored
            # there, and a later region holding the next site (where the deletion prints); the same with rows below it
            SL = K["SEL_LAST_ROWS"]
            e_ = batch.ref_end()
            regs = [(b - 1, e - 1) for _, b, e in case["regions"]]

            def anchored(a, rows_ok):
                cov = [i for i in range(batch.n_reads) if batch.pos[i] <= a < e_[i]]
                dels = [i for i in cov if facts[i]["ops"][0][1] == "M" and facts[i]["ops"][1][1] == "D"
                        and batch.pos[i] + facts[i]["ops"][0][0] - 1 == a]
                ends_region = [k for k, (b, e) in enumerate(regs) if e == a]
                later = ends_region and any(b <= a + 1 <= e for b, e in regs[ends_region[0] + 1:])
                return bool(cov) and all(batch.lib[i] != 0xFFFF and rows_ok(int(batch.lib[i])) for i in cov) and bool(dels) and bool(later)
            _both(all(anchored(a, lambda r: r < SL) for a in case["probe"]["low_anchors"]),
                  all(anchored(a, lambda r: r >= SL) for a in case["probe"]["anchors"]) and len(case["lib_names"]) > SL + 4, target)
        elif target == "cigar_stage":
            ch = [c for c in k1_chunks(batch, tile_ranges(batch, first_pos, end)) if c["r1"] - c["r0"] == K["STAGE_READS"]]
            _both(any(c["cstaged"] and c["cops"] > K["STAGE_CIGAR"] - 8 for c in ch),
                  any(not c["cstaged"] and c["cops"] <= K["STAGE_CIGAR"] + 8 for c in ch), target)
        elif target in ("ncover_8bit", "clip_sum_16bit", "se_sum_16bit", "mmq_sum_16bit"):
            s = site_sums(batch, facts, first_pos, end)
            key, lim = {"ncover_8bit": ("depth", 255), "clip_sum_16bit": ("clip", 0xFFFF), "se_sum_16bit": ("se", 0xFFFF),
                        "mmq_sum_16bit": ("mmq", 0xFFFF)}[target]
            v = s[key]
            _both(lim in v and lim - 1 in v if key == "depth" else lim in v, lim + 1 in v, target)
            if key == "se":
                assert (v > 0xFFFFFFFF - 0x10000).any(), "se_sum_16bit: no site whose SE sum wraps below zero"
        elif target == "deep_block":
            counts = []
            for (ci2, b, e) in case["regions"]:
                if e - b + 1 <= 2:
                    _, bg, en, sub = cases.region_reads(case, ci2, b, e)
                    counts.append(sub.n_reads)
            D = K["DEEP_THREADS"]
            _both(D - 1 in counts and D in counts, D + 1 in counts, target)
        elif target == "icache":
            C = K["DEEP_ICACHE"]
            per_site = {}      # distinct short insertion alleles (the inserted nibbles) per anchor site
            so = batch.seq_off.astype(np.int64)
            for i, f in enumerate(facts):
                ops = f["ops"]
                if len(ops) == 3 and ops[1][1] == "I" and ops[1][0] <= 3:
                    pk = batch.seq[so[i]:so[i + 1]]
                    nib = np.empty(pk.shape[0] * 2, np.uint8); nib[0::2] = pk >> 4; nib[1::2] = pk & 15
                    per_site.setdefault(int(batch.pos[i]) + ops[0][0] - 1, set()).add(tuple(nib[ops[0][0]:ops[0][0] + ops[1][0]].tolist()))
            ns = [len(v) for v in per_site.values()]
            _both(C in ns, C + 1 in ns, target)
        elif target == "indel_len":
            ins = {l for f in facts for l, o in f["ops"] if o == "I"}
            dels = {l for f in facts for l, o in f["ops"] if o == "D"}
            _both(8 in ins and 127 in dels, 9 in ins and 128 in dels, target)
        elif target == "byte_values":
            _both(bool((batch.qual == 0xFF).any()), bool((batch.mapq == 255).any()), target)
        else:
            raise AssertionError(f"unknown target {target}")


CASES = boundary_cases.all_cases()


def test_kernel_constants_parse():
    K = kernel_constants()
    assert set(CONST_NAMES) <= set(K)
    assert K["STAGE_QUAL"] == K["STAGE_READS"] * 152 + 32 and K["K0_QUAL_CAP"] == K["K0_READS"] * 160 + 32


@pytest.mark.parametrize("case", CASES + (boundary_cases.queue_rows(),), ids=[c["name"] for c in CASES] + ["queue_rows"])
def test_case_straddles_its_limits(case):
    check_targets(case)


def test_cases_cover_every_window_start_and_contig_length_residue():
    wins = {c["contigs"][0][3] for c in CASES if c["name"].startswith("refwin")}
    lens = {c["contigs"][0][1] % 4 for c in CASES if c["name"].startswith("refwin")}
    assert wins == {0, 1, 4095, 4097} and lens == {0, 1, 2, 3}
    # reads run to and past the contig end
    for c in CASES:
        if c["name"].startswith("refwin"):
            assert (c["batch"].ref_end() > c["contigs"][0][1]).any()


JOBS = boundary_cases.jobs()


@pytest.mark.parametrize("job", JOBS, ids=[j[4] for j in JOBS])
def test_oracle_equals_reference_binary_on_boundary_cases(job):
    case, fname, fl, sl, key = job
    cases.assert_anchor("boundary_sha256.json", key, cases.run_oracle(case, fl, site_list=sl).text)


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("job", JOBS, ids=[j[4] for j in JOBS])
def test_engine_equals_oracle_on_boundary_cases(job, monkeypatch):
    case, fname, fl, sl, key = job
    want = cases.run_oracle_cached(case, fl, sl)
    cases.assert_same(cases.run_engine(case, fl, site_list=sl), want)
    if len(case["regions"]) == 1 and "max_cnt" not in fl:
        # the copy path (run_engine's one push is the pipelined path)
        cases.assert_same(cases.run_engine(case, fl, site_list=sl, dump=False, push="halves"), want, "two pushes",
                          fields=("text", "warnings"))
    if sl:
        monkeypatch.setenv("BRC_DEEP_MIN_READS", "1")
        cases.assert_same(cases.run_engine(case, fl, site_list=sl), want, "deep-forced")


def test_fastmath_selftest_bound_covers_every_hot_numerator():
    """The self-test's numerator loop reaches 2 FASTDIV_MAX + 2 for every divisor: the hot path forms up to 2 (l_qseq - 1)."""
    K = kernel_constants()
    src = open(os.path.join(CSRC, "brc_kernels.cu")).read()
    body = src[src.index("fastmath_selftest_kernel("):]
    m = re.search(r"for\s*\(\s*int\s+a\s*=\s*threadIdx\.x\s*;\s*a\s*<=\s*([^;]+);", body)
    assert m, "numerator loop of fastmath_selftest_kernel not found"
    # the loop's bound for the smallest divisor must reach every numerator the hot path forms
    assert eval(m.group(1), {}, dict(K, b=1)) >= 2 * K["FASTDIV_MAX"] + 2


@pytest.mark.gpu
def test_fastmath_selftest_covers_every_hot_numerator():
    """brc_selftest_fastmath checks div_small against __fdiv_rn for every divisor b <= FASTDIV_MAX and every numerator up to
    2 FASTDIV_MAX + 2; a wrong quotient anywhere fails it."""
    from bam_readcount_b200.engine import Engine
    e = Engine()
    try:
        assert e.lib.brc_selftest_fastmath(e.h, kernel_constants()["FASTDIV_MAX"]) == 0
    finally:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [dict(), dict(per_lib=True)], ids=["alllib", "perlib"])
def test_secondary_pool_grows_and_stays_exact(flags):
    case = pool_case()
    want = cases.run_oracle(case, flags, site_list=True)
    # pipelined path (one borrowed push): its overflow falls through to the plain path, which grows the pool
    got = cases.run_engine(case, flags, site_list=True)
    n_slots = cases.region_geometry(case, case["regions"][0])[5]
    assert got.n_sec > initial_pool_cap(case, flags, n_slots), "the pool never outgrew its initial capacity: no retry ran"
    cases.assert_same(got, want, fields=("dump", "text"))
    t2 = cases.run_engine(case, flags, site_list=True, dump=False, push="halves").text      # copy path
    assert t2 == want.text, first_diff(t2, want.text)
    for mc, mf in THRESHOLDS:                                  # filtered path
        text = cases.run_engine(case, flags, True, site_filter=(mc, mf)).text
        assert text == select_lines(want.text, mc, mf), (mc, mf)


@pytest.mark.gpu
@pytest.mark.parametrize("which", [0, 1], ids=["300k_sites", "40_libraries"])
def test_site_selection_at_scale(which):
    """More than 1024 scan partials (> 262 144 sites) with adjacent and overlapping argv regions; and -p with 40 libraries and
    library-less reads over 300 adjacent argv regions (the LIBRARY_UNAVAILABLE count of the selection's site pass).  That the
    deletion queue survives rows >= SEL_LAST_ROWS is test_site_selection_ships_the_queue_of_high_library_rows's."""
    K = kernel_constants()
    case = selection_cases()[which]
    flags = dict(per_lib=True) if which == 1 else dict()
    if which == 0:
        assert case["regions"][0][2] - case["regions"][0][1] + 1 > 1024 * K["SCAN_CTA"]
    else:
        assert len(case["lib_names"]) > K["SEL_LAST_ROWS"]
    otext, _, owarn = cases.run_oracle(case, flags, site_list=False)
    for mc, mf in THRESHOLDS:
        got = cases.run_engine(case, flags, False, site_filter=(mc, mf))
        want = select_lines(otext, mc, mf)
        assert got.text == want, (mc, mf, first_diff(got.text, want))
        if which == 1:
            assert owarn[2] > 0 and got.warnings[3] == owarn[2], (got.warnings, owarn)


@pytest.mark.gpu
def test_site_selection_ships_the_queue_of_high_library_rows():
    """boundary_cases.queue_rows: deletions of library rows >= SEL_LAST_ROWS anchored at an argv region's last site, a site no lower
    row covers and whose line fails the filter.  They print only in the next region, from the never-cleared deletion queue, so the
    selection must ship that site for those rows (sel_site_kernel's global reg_last branch); rows < 32 go through shared memory."""
    case = boundary_cases.queue_rows()
    flags = dict(per_lib=True)
    want_all = cases.run_oracle(case, flags, site_list=False)
    cases.assert_same(cases.run_engine(case, flags, site_list=False, dump=False), want_all, fields=("text", "warnings"))
    for a in case["probe"]["anchors"]:                          # the carried deletions do print in the next region
        assert any(ln.startswith(f"c\t{a + 2}\t") and "\t-" in ln for ln in want_all.text.splitlines()), a
    for mc, mf in THRESHOLDS:
        text = cases.run_engine(case, flags, False, site_filter=(mc, mf)).text
        want = select_lines(want_all.text, mc, mf)
        assert text == want, (mc, mf, first_diff(text, want))


@pytest.mark.gpu
def test_device_path_reports_pool_overflow_and_is_exact_when_replanned():
    """brc_plan_device with a secondary pool of 1024 records on the random-base pool case: brc_fetch_device_results must return
    BRC_E_OVERFLOW (the device path has no retry).  Re-planned with room, every raw accumulator equals the oracle's."""
    import torch
    from bam_readcount_b200.engine import BrcError, admitted
    case = pool_case()
    odump = cases.run_oracle(case, dict(), site_list=True).dump
    region = case["regions"][0]
    tid, _, _, sub = cases.region_reads(case, *region)
    assert len(admitted(sub, tid, 10_000_000)) == sub.n_reads        # the device path admits every read it is given
    dev = torch.device("cuda", 0)
    cb, keep = cases.device_batch(sub, dev)
    with cases.open_engine(case) as e:
        s = torch.cuda.Stream(device=dev)
        with pytest.raises(BrcError) as err:
            cases.run_device(e, case, region, cb, s, n_sec_cap=1024)
        assert err.value.status == -8          # BRC_E_OVERFLOW
        edump = cases.run_device(e, case, region, cb, s)
        assert edump == odump, first_diff(edump, odump)
    del keep


@pytest.mark.gpu
def test_bgzf_record_scan_over_more_than_one_scan_level():
    """A synth_cb sample of 1500 blocks decoded on the device as ONE span: its record framing runs the shared exclusive scan over
    more than 1024 partials (> 262 144 records).  Every array equals bamio's host decode."""
    import tempfile
    from bam_readcount_b200 import bamio, synth_cb
    from bam_readcount_b200.engine import Engine
    samtools = cases.samtools()
    tmp = tempfile.mkdtemp()
    sp = synth_cb.Spec(seed=31, contig_len=1280 * 1600)
    info = synth_cb.write_sample_bam(sp, 0, 0, 1500, tmp, samtools)
    hdr, host = bamio.read_bam(info["bam"])
    rg_lib = {rg: hdr.lib_of_rg(rg) for rg in hdr.rg_lb}
    span = bamio.bam_span(info["bam"], bamio.BaiIndex(info["bam"] + ".bai"), 0, 0, info["length"], rg_lib)
    e = Engine(per_lib=True, lib_names=hdr.lib_names)
    try:
        got = e.decode_bam_span(span)
    finally:
        e.close()
    K = kernel_constants()
    assert got.n_reads > 1024 * K["SCAN_CTA"]
    want = host.select(host.fetch(0, 0, info["length"]))
    assert got.n_reads == want.n_reads == host.n_reads
    for k in ("pos", "flag", "mapq", "lib", "l_qseq", "nm", "sm", "cigar_off", "cigar", "seq_off", "seq", "qual_off", "qual"):
        g, w = np.asarray(getattr(got, k)), np.asarray(getattr(want, k))
        assert g.shape == w.shape and np.array_equal(g, w.astype(g.dtype)), k
