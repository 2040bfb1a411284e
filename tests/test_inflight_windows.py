"""The records bench.py's timed loops compute with every engine handle in flight, read from those loops as they run.

The C4 loop runs three WindowRunners round-robin with no host wait between windows (a runner waits only for its own previous
window), shares contig references between them and mixes resident and regenerated windows; C3 queues runs back to back on one
planned handle; C5 alternates deep launches between two handles.  Each test drives a loop with bench.py's calls in bench.py's
order and takes every window's records with ``inflight_cases.Capture`` (gather_round's ordering: wait for `done`, copy, record
`sent`), then checks them:
  * C4, 3 contigs x 6 windows of 100 blocks, -i / -q 20 -b 20 / -p with 8 libraries, two passes: every window equals a serial
    run of it on a fresh runner bit for bit, and the serial run equals the oracle over the whole window;
  * C4 at its real geometry (12.5 Mb windows, 2 contigs of 10): checksums of the words and a digest of the pool equal a serial
    run's, and one 20 000-site range of each capture equals the oracle;
  * C3: 4 runs queued behind one another equal each other and the oracle; with a site filter, each run selects the rule's lines;
  * C5: 6 deep launches on two handles equal serial runs and the oracle at every site;
  * first use in a fresh process: two threads whose first runs build the per-device tables give what runs one after the other give.
Each test also asserts that it reached the in-flight path: windows of different runners overlapped on the GPU, two contigs were
live at once, resident and regenerated windows both ran, C3's runs were all queued before the first one finished.
"""
from __future__ import annotations

import os
import subprocess
import sys

import numpy as np
import pytest

import inflight_cases as ic
from bam_readcount_b200 import stream as st
from bam_readcount_b200 import synth_cb as sc
from cases import ROOT

C4_FLAG_SETS = {
    "ic": (dict(insertion_centric=True), []),                 # C4's own flags
    "q20b20": (dict(min_mapq=20, min_bq=20), []),
    "perlib": (dict(per_lib=True), ic.LIBS),
}


def _resident_small(k: int) -> bool:
    return k % 2 == 0


def _resident_real(k: int) -> bool:
    return k % 4 == 0


# ------------------------------------------------------------------------------------------------ CPU
def test_small_schedule_changes_contig_while_another_runner_holds_the_last():
    """The small C4 geometry deals windows so that a runner moves to the next contig while the other two still read the one it
    left (windows 6 and 7), again at the next contig (12, 13), and from the last contig back to the first when the second pass
    starts (18, 19); every runner runs resident and regenerated windows.  The real geometry changes contig in flight too."""
    spec = sc.Spec(**ic.SMALL_SPEC)
    wins = st.wgs_windows(spec, ic.SMALL_WINDOWS_PER_CONTIG)
    assert len(wins) == 18 and all(w.blk_hi - w.beg // sc.BLOCK_BP == 100 for w in wins)
    order = ic.deal(len(wins))
    assert ic.contig_changes_in_flight(wins, order, passes=2) == [6, 7, 12, 13, 18, 19, 24, 25, 30, 31]
    for r in range(ic.N_RUNNERS):
        mine = [k for k in range(len(wins)) if order[k] == r]
        assert any(_resident_small(k) for k in mine) and not all(_resident_small(k) for k in mine)
    real = st.wgs_windows(sc.Spec(**ic.REAL_SPEC), ic.REAL_WINDOWS_PER_CONTIG)
    assert len(real) == 20 and real[0].n_sites == 9766 * sc.BLOCK_BP
    assert ic.contig_changes_in_flight(real, ic.deal(len(real))) == [10, 11]


def test_packed_view_restatement_chains_every_key():
    """results_from_packed, which turns captured records into the dump's view, on hand-made records: keys chain per (row, slot),
    escaped sites take their record, slot_range re-addresses a range's records."""
    n_rows, n_slots = 2, 5
    words = np.zeros((8, n_rows, n_slots), dtype=np.uint32)
    words[0, 0, 1] = 3 | 3 << 8 | 2 << 16 | 1 << 24
    words[1, 0, 1] = 1                                             # primary base A
    words[1, 1, 3] = 7                                             # escaped
    sec = np.zeros((4, 18), dtype=np.uint32)
    sec[0, 0], sec[0, 2], sec[0, 5] = 1, 6 | 2 << 8, 1              # insertion of length 2 at (row 0, slot 1)
    sec[1, 0], sec[1, 2], sec[1, 5] = 1, 2, 1                       # base C at (row 0, slot 1)
    sec[2, 0], sec[2, 2], sec[2, 4], sec[2, 5] = n_slots + 3, 8 + 4 | 300 << 8, 299, 300   # escaped G site at (row 1, slot 3)
    sec[3, 0], sec[3, 2], sec[3, 5] = n_slots + 4, 7 | 1 << 8, 1    # deletion at (row 1, slot 4)
    r = ic.results_from_packed(words, sec, [dict(tid=0, beg=0, end=n_slots, site_list_mode=0, read_lo=0, read_hi=0, slot_base=0,
                                                 first_pos=0, n_slots=n_slots)])
    chain = []
    j = int(r.sec_head[0, 1])
    while j >= 0:
        chain.append(j)
        j = int(r.sec_next[j])
    assert sorted(chain) == [0, 1] and int(r.sec_head[1, 4]) == 3 and int(r.sec_head[1, 3]) == -1
    assert r.ncover[1, 3] == 300 and r.npass[1, 3] == 299 and r.pbase[1, 3] == 4 and r.sec_kind[2] == 0xFF
    assert r.ncover[0, 1] == 3 and r.pbase[0, 1] == 1 and r.pstats[0, 0, 1] == 2
    sub = ic.slot_range(words, sec, 1, 4, n_slots)
    assert sub[:, 0].tolist() == [0, 0, 3 + 2]


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def oracle_pool():
    """Worker processes for the oracle comparisons (the Python dump of a window takes seconds); joined when the module ends."""
    import multiprocessing as mp
    from concurrent.futures import ProcessPoolExecutor
    with ProcessPoolExecutor(max_workers=max(1, min(8, os.cpu_count() or 1)), mp_context=mp.get_context("spawn")) as ex:
        yield ex


def _failures(futures):
    return [m for m in (f.result(timeout=1800) for f in futures) if m]


class _Spans:
    """A timed event at the start and at the end of each window on its runner's stream."""

    def __init__(self):
        self.items = []

    def start(self, stream):
        import torch
        ev = torch.cuda.Event(enable_timing=True)
        ev.record(stream)
        return ev

    def end(self, who, ev0, stream):
        ev1 = self.start(stream)
        self.items.append((who, ev0, ev1))

    def overlaps(self):
        """Pairs of windows of different runners whose spans overlapped on the GPU (call after a synchronize)."""
        t0 = self.items[0][1]
        sp = [(who, t0.elapsed_time(a), t0.elapsed_time(b)) for who, a, b in self.items]
        return [(i, j) for i in range(len(sp)) for j in range(i + 1, len(sp))
                if sp[i][0] != sp[j][0] and sp[i][1] < sp[j][2] and sp[j][1] < sp[i][2]]


def _run_c4(runners, wins, resident, cap, passes, spans, gate):
    """bench.py's one_pass with one runner per window round-robin, `passes` times; window j of the run is captured as j.
    gate: hold the stream of the runner that generates a contig (the first to move to it) before its window, so the runners
    that follow it onto the contig queue their windows while the reference is not ready yet, and must wait for it."""
    live, kinds = 0, set()
    for p in range(passes):
        for k, w in enumerate(wins):
            run = runners[k % len(runners)]
            ev0 = spans.start(run.stream)
            if gate and w.contig != run.cur_contig and w.contig not in run.refs.live():
                ic.hold(run.stream)
            run.launch(w, resident=resident.get(k))
            spans.end(k % len(runners), ev0, run.stream)
            cap.take(p * len(wins) + k, run.eng, run.done, run.sent)
            live = max(live, len(run.refs.live()))
            kinds.add(k in resident)
    return live, kinds


def _prefill(spec, wins, which, device):
    """Resident windows, filled before the loop with one shared scratch, as bench.py keeps them."""
    import torch
    max_reads = max(spec.window_reads(w.blk_lo, w.blk_hi) for w in wins)
    scratch = torch.empty(max_reads // sc.BLOCK_READS + 4, dtype=torch.int64, device=device)
    out = {}
    for k, w in enumerate(wins):
        if which(k):
            out[k] = sc.DeviceWindow(spec, spec.window_reads(w.blk_lo, w.blk_hi), device, scratch=scratch, with_region=False)
            out[k].fill(w.contig, w.blk_lo, w.blk_hi, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("fname", list(C4_FLAG_SETS))
def test_c4_loop_windows_equal_serial_runs_and_the_oracle(fname, oracle_pool):
    """Three runners, 18 windows on 3 contigs, half of them resident, two passes: every captured window equals a serial run of
    it on a fresh runner (packed words and sorted pool records), and each serial run's dump over the whole window equals the
    oracle's (bench.py's oracle_dump recipe).  The runner that generates a contig is held back before that window
    (inflight_cases.hold), so the windows the other runners queue on that contig wait for its reference on the GPU."""
    import torch
    flags, libs = C4_FLAG_SETS[fname]
    dev = torch.device("cuda", 0)
    spec = sc.Spec(**ic.SMALL_SPEC)
    wins = st.wgs_windows(spec, ic.SMALL_WINDOWS_PER_CONTIG)
    rows = len(libs) if flags.get("per_lib") else 1
    max_reads = max(spec.window_reads(w.blk_lo, w.blk_hi) for w in wins)
    passes = 2
    runners = [st.WindowRunner(spec, max_reads, dev, flags, libs) for _ in range(ic.N_RUNNERS)]
    try:
        resident = _prefill(spec, wins, _resident_small, dev)
        cap = ic.Capture(dev, [ic.window_geometry(rows, w) for w in wins] * passes)
        spans = _Spans()
        live, kinds = _run_c4(runners, wins, resident, cap, passes, spans, gate=True)
        torch.cuda.synchronize()
        overlaps = spans.overlaps()
        captured = [cap.host(j, rows) for j in range(passes * len(wins))]
        del cap, resident
    finally:
        for r in runners:
            r.close()
    assert overlaps, "no two windows of different runners overlapped on the GPU"
    assert live >= 2, "never more than one contig live"
    assert kinds == {True, False}, "resident and regenerated windows did not both run"

    # serial: a fresh runner (and a Spec object of its own, so its contig references are not the loop's), one window at a time
    spec2 = sc.Spec(**ic.SMALL_SPEC)
    serial = st.WindowRunner(spec2, max_reads, dev, flags, libs)
    futures, diffs = [], []
    try:
        for k, w in enumerate(wins):
            serial.busy = False
            serial.launch(w)
            torch.cuda.synchronize()
            res = serial.eng.fetch_device_results(serial.stream.cuda_stream)
            pk = serial.eng.packed()
            for p in range(passes):
                d = ic.diff_packed(f"{fname} pass {p + 1} window {k} (runner {k % ic.N_RUNNERS}, contig {w.contig}, "
                                   f"{'resident' if _resident_small(k) else 'regenerated'})", captured[p * len(wins) + k],
                                   (pk.words, pk.sec), w.first_pos)
                if d:
                    diffs.append(d)
            futures.append(oracle_pool.submit(ic.check_window_against_oracle, f"{fname} serial window {k}", ic.SMALL_SPEC, flags, libs,
                                              w.contig, w.first_pos, w.end, w.blk_lo, res))
    finally:
        serial.close()
    assert not diffs, "\n".join(diffs[:6])
    bad = _failures(futures)
    assert not bad, "\n".join(bad[:4])


@pytest.mark.gpu
def test_c4_loop_at_real_geometry(oracle_pool):
    """C4's own geometry: 12.5 Mb windows (9766 blocks), 10 per 125 Mb contig, 2 contigs, -i, three runners for one pass, every
    fourth window resident; the runner that takes window 10 moves to contig 1 while the other two still read contig 0.  Each
    capture holds a checksum of the window's 400 MB of words, its whole pool and one 20 000-site range of its words; they equal
    a serial run's (the pools by an order-independent digest), and the range equals the oracle.  Device memory in use at the
    peak, against what was free before: 12.5 GB measured on an H100 80GB HBM3 (three runners, five resident windows, 20 pool
    copies), where the C4 bench on one H100 fills all but 14 GB of the 80 GB with resident windows."""
    import torch
    flags = dict(insertion_centric=True)
    dev = torch.device("cuda", 0)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(dev)[0]
    spec = sc.Spec(**ic.REAL_SPEC)
    wins = st.wgs_windows(spec, ic.REAL_WINDOWS_PER_CONTIG)
    max_reads = max(spec.window_reads(w.blk_lo, w.blk_hi) for w in wins)
    rng = np.random.default_rng(77)
    span = 20_000
    ranges, lo = [], []
    for w in wins:
        a = int(rng.integers(w.first_pos, w.end - span))
        lo.append(a)
        ranges.append((a - w.first_pos, a - w.first_pos + span, 1, w.n_slots))
    runners = [st.WindowRunner(spec, max_reads, dev, flags) for _ in range(ic.N_RUNNERS)]
    try:
        resident = _prefill(spec, wins, _resident_real, dev)
        cap = ic.Capture(dev, [ic.window_geometry(1, w) for w in wins], ranges)
        spans = _Spans()
        live, kinds = _run_c4(runners, wins, resident, cap, 1, spans, gate=False)
        torch.cuda.synchronize()
        used_gb = (free0 - torch.cuda.mem_get_info(dev)[0]) / 1e9
        overlaps = spans.overlaps()
        del resident
    finally:
        for r in runners:
            r.close()
    print(f"\nC4 real geometry: {used_gb:.1f} GB of device memory in use at the peak")
    assert overlaps and live >= 2 and kinds == {True, False}, (len(overlaps), live, kinds)
    assert used_gb < 30, f"{used_gb:.1f} GB in use"

    spec2 = sc.Spec(**ic.REAL_SPEC)
    serial = st.WindowRunner(spec2, max_reads, dev, flags)
    acc = torch.zeros(1, dtype=torch.int64, device=dev)
    futures, diffs = [], []
    try:
        for k, w in enumerate(wins):
            serial.busy = False
            serial.launch(w)
            torch.cuda.synchronize()
            words, secb = serial.packed_tensors()
            acc.zero_()
            sc.checksum_device(words, acc, torch.cuda.current_stream().cuda_stream)
            want_sec = secb.cpu().numpy().view(np.uint32).reshape(-1, 18)
            got_words, got_sec = cap.host(k, 1)
            what = f"window {k} (runner {k % ic.N_RUNNERS}, contig {w.contig}, {'resident' if _resident_real(k) else 'regenerated'})"
            if int(acc.item()) != int(cap.checksum[k].item()):
                diffs.append(f"{what}: words checksum differs from the serial run's")
            if len(got_sec) != len(want_sec):
                diffs.append(f"{what}: {len(got_sec)} pool records, the serial run has {len(want_sec)}")
            elif not np.array_equal(ic.record_digest(got_sec), ic.record_digest(want_sec)):
                diffs.append(f"{what}: pool records differ from the serial run's")
            s0, s1 = ranges[k][0], ranges[k][1]
            sub = ic.slot_range(got_words, got_sec, s0, s1, w.n_slots)
            res = ic.results_from_packed(got_words, sub, [dict(tid=w.contig, beg=w.beg, end=w.end, site_list_mode=0, read_lo=0,
                                                                read_hi=0, slot_base=0, first_pos=lo[k], n_slots=span)])
            futures.append(oracle_pool.submit(ic.check_window_against_oracle, f"{what} sites [{lo[k]}, {lo[k] + span})", ic.REAL_SPEC,
                                              flags, [], w.contig, lo[k], lo[k] + span, w.blk_lo, res))
    finally:
        serial.close()
    del cap
    assert not diffs, "\n".join(diffs[:6])
    bad = _failures(futures)
    assert not bad, "\n".join(bad[:4])


def _oracle_text(spec, flags, w):
    """The oracle's text of window w as one argv region."""
    from oracle.oracle import Oracle
    hb, _ = spec.window_host(w.contig, w.blk_lo, w.blk_hi)
    o = Oracle(**flags)
    o.region(hb.select(hb.fetch(w.contig, w.first_pos, w.end)), tid=w.contig, beg=w.beg, end=w.end, contig=f"chr{w.contig + 1}",
             chrom_len=spec.contig_len, ref_seq=spec.ref_host(w.contig, 0, spec.contig_len), ref_win_beg=0, site_list_mode=False)
    return o.text()


@pytest.mark.gpu
def test_c3_loop_back_to_back_runs(oracle_pool):
    """C3's loop on a 1 Mb contig, -q 20 -b 20: one planned handle, its window resident, 4 run_device calls queued on the
    runner's stream, each behind wait_event(sent), a capture after each.  A spin kernel at the head of the stream holds the runs
    back, so the host must have queued all four before the first finishes: no call of the loop may wait on the stream.  All four
    captures are identical and equal the oracle.  Then, with the reference's characters on the host and a site filter of 2 reads,
    4 runs back to back on the same plan, each fetched before the next is queued: every run's emit-1 sites are exactly the
    lines site_filter_rule keeps from the oracle's text."""
    import torch
    from site_filter_rule import select_lines
    flags = dict(min_mapq=20, min_bq=20)
    dev = torch.device("cuda", 0)
    spec_kw = dict(seed=1234, contig_len=782 * sc.BLOCK_BP, n_contigs=1)
    spec = sc.Spec(**spec_kw)
    w = st.wgs_windows(spec, 1)[0]
    run = st.WindowRunner(spec, spec.window_reads(w.blk_lo, w.blk_hi), dev, flags)
    n_runs = 4
    try:
        sp = run.stream.cuda_stream
        run._ensure_reference(w.contig)                  # launch()'s set-up without its run: the plan, the window resident
        n = run.dw.fill(w.contig, w.blk_lo, w.blk_hi, sp)
        reg = st.window_region(w)
        reg.read_hi = n
        run.eng.plan_device([reg], n, 0)
        torch.cuda.synchronize()
        cap = ic.Capture(dev, [ic.window_geometry(1, w)] * n_runs)
        ends = []
        ic.hold(run.stream)
        for i in range(n_runs):
            run.stream.wait_event(run.sent)
            run.eng.run_device(run.dw.c_batch(), None, sp)
            with torch.cuda.stream(run.stream):
                run.done.record(run.stream)
                ends.append(torch.cuda.Event())
                ends[-1].record(run.stream)
            cap.take(i, run.eng, run.done, run.sent)
        first_pending = not ends[0].query()
        torch.cuda.synchronize()
        captured = []
        for i in range(n_runs):
            captured.append(cap.host(i, 1, f"run {i + 1}"))
            d = ic.diff_packed(f"run {i + 1} against run 1", captured[i], captured[0], w.first_pos)
            assert not d, d
        assert first_pending, "run 1 had finished before the host queued run 4"

        # with a site filter: the reference's characters on the host too, so the device and the rule judge the same bases
        run.eng.set_reference(w.contig, f"chr{w.contig + 1}", spec.contig_len, spec.ref_host(w.contig, 0, spec.contig_len), 0)
        run.eng.set_site_filter(2)
        selected = []
        for i in range(n_runs):
            run.stream.wait_event(run.sent)
            run.eng.run_device(run.dw.c_batch(), None, sp)
            with torch.cuda.stream(run.stream):
                run.done.record(run.stream)
            with torch.cuda.stream(cap.stream):
                cap.stream.wait_event(run.done)
                assert run.eng.fetch_device_results(cap.stream.cuda_stream) is None
                selected.append([p + 1 for p in run.eng.selected().positions(1)])
                run.sent.record(cap.stream)
        torch.cuda.synchronize()
    finally:
        run.close()
    region = dict(tid=w.contig, beg=w.beg, end=w.end, site_list_mode=0, read_lo=0, read_hi=n, slot_base=0, first_pos=w.first_pos,
                  n_slots=w.n_slots)
    res = ic.results_from_packed(*captured[0], [region])
    fut = oracle_pool.submit(ic.check_window_against_oracle, "run 1", spec_kw, flags, [], w.contig, w.first_pos, w.end, w.blk_lo, res)
    want = [int(ln.split("\t")[1]) for ln in select_lines(_oracle_text(spec, flags, w), 2).splitlines()]
    assert len(want) > 100
    for i, got in enumerate(selected):
        if got != want:
            extra, missing = sorted(set(got) - set(want)), sorted(set(want) - set(got))
            raise AssertionError(f"filtered run {i + 1}: {len(got)} sites selected, the rule keeps {len(want)}; "
                                 f"first extra {extra[:3]}, first missing {missing[:3]} (1-based)")
    bad = _failures([fut])
    assert not bad, bad[0]


@pytest.mark.gpu
def test_c5_loop_two_handles(oracle_pool):
    """C5's loop: DEEP spec, 8 libraries, 3000 reads per site, 6 sites per launch, 6 launches alternating between two handles on
    two streams, -p -d 100000000, two launches resident.  The capture releases a handle (`sent`) and the next launch on it
    waits for that as for its kernels.  Every launch's capture equals a serial run, and every site of it equals the oracle."""
    import torch
    from bam_readcount_b200.engine import CRegion, Engine
    from oracle.oracle import Oracle
    flags = dict(per_lib=True, max_cnt=100_000_000)
    spec_kw = dict(seed=1234, mode=sc.DEEP, n_libs=8, depth=3000, site_stride=1000, n_sites=36, contig_len=sc.BLOCK_BP)
    spec = sc.Spec(**spec_kw)
    dev = torch.device("cuda", 0)
    per, depth = 6, spec.depth
    wins = [(a, a + per) for a in range(0, spec.n_sites, per)]
    L = spec.deep_contig_len()

    def regions_of(a, b):
        return [CRegion(0, spec.site_pos(k), spec.site_pos(k) + 1, 1, (k - a) * depth, (k - a + 1) * depth, 2 * (k - a),
                        spec.site_pos(k) - 1, 2) for k in range(a, b)]

    def region_dicts(a, b):
        return [dict(tid=g.tid, beg=g.beg, end=g.end, site_list_mode=g.site_list_mode, read_lo=g.read_lo, read_hi=g.read_hi,
                     slot_base=g.slot_base, first_pos=g.first_pos, n_slots=g.n_slots) for g in regions_of(a, b)]

    ref_ascii = torch.empty(L + 64, dtype=torch.uint8, device=dev)
    import ctypes as C
    sc.load().brc_synth_ref_device(C.byref(spec.c), 0, 0, L, ref_ascii.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    engs = [Engine(device=0, lib_names=ic.LIBS, **flags) for _ in range(2)]
    try:
        dws = [sc.DeviceWindow(spec, per * depth, dev) for _ in range(2)]
        resident = {}
        for i in (0, 3):
            a, b = wins[i]
            resident[i] = sc.DeviceWindow(spec, (b - a) * depth, dev, scratch=dws[0].t["scratch"], with_region=True)
            resident[i].fill(0, a, b, torch.cuda.current_stream().cuda_stream)
        streams = [torch.cuda.Stream(device=dev) for _ in range(2)]
        done = [torch.cuda.Event() for _ in range(2)]
        sent = [torch.cuda.Event() for _ in range(2)]
        for e in engs:
            e.set_reference_device(0, "chr1", L, 0, ref_ascii.data_ptr(), L, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        cap = ic.Capture(dev, [(8 * 2 * per * 4 * 8, 65536)] * len(wins))
        spans = _Spans()
        used = [False, False]
        for i, (a, b) in enumerate(wins):                  # bench.py's run_deep launch(), the capture's release added
            h = i % 2
            if used[h]:
                done[h].synchronize()
                sent[h].synchronize()
            s = streams[h]
            ev0 = spans.start(s)
            if not used[h]:
                ic.hold(s)                                 # the first launches of both handles are queued together
            dw = resident.get(i)
            if dw is None:
                dw = dws[h]
                dw.fill(0, a, b, s.cuda_stream)
            engs[h].plan_device(regions_of(a, b), (b - a) * depth, 65536)
            engs[h].run_device(dw.c_batch(), dw.t["region"].data_ptr(), s.cuda_stream)
            with torch.cuda.stream(s):
                done[h].record(s)
            spans.end(h, ev0, s)
            used[h] = True
            cap.take(i, engs[h], done[h], sent[h])
        torch.cuda.synchronize()
        overlaps = spans.overlaps()
        captured = [cap.host(i, 8, f"launch {i}") for i in range(len(wins))]
    finally:
        for e in engs:
            e.close()
    assert overlaps, "no two launches of the two handles overlapped on the GPU"

    ref = spec.ref_host(0, 0, L)
    serial = Engine(device=0, lib_names=ic.LIBS, **flags)
    try:
        serial.set_reference_device(0, "chr1", L, 0, ref_ascii.data_ptr(), L, torch.cuda.current_stream().cuda_stream)
        dw = sc.DeviceWindow(spec, per * depth, dev)
        s = torch.cuda.Stream(device=dev)
        for i, (a, b) in enumerate(wins):
            dw.fill(0, a, b, s.cuda_stream)
            serial.plan_device(regions_of(a, b), (b - a) * depth, 65536)
            serial.run_device(dw.c_batch(), dw.t["region"].data_ptr(), s.cuda_stream)
            serial.fetch_device_results(s.cuda_stream)
            pk = serial.packed()
            d = ic.diff_packed(f"launch {i} (handle {i % 2}, sites {a}..{b - 1})", captured[i], (pk.words, pk.sec), 0)
            assert not d, d
            res = ic.results_from_packed(*captured[i], region_dicts(a, b))
            hb, _ = spec.window_host(0, a, b)
            for k in range(a, b):
                p = spec.site_pos(k)
                o = Oracle(lib_names=ic.LIBS, **flags)
                o.region(hb, tid=0, beg=p, end=p + 1, contig="chr1", chrom_len=L, ref_seq=ref, ref_win_beg=0, site_list_mode=True,
                         read_lo=(k - a) * depth, read_hi=(k - a + 1) * depth)
                ed = res.dump_range(hb, {0: (0, ref)}, k - a, p - 1, p + 1)
                assert ed == o.dump(), f"launch {i}, site {k} (position {p})"
    finally:
        serial.close()


FIRST_USE = r"""
import sys, threading
import numpy as np
from bam_readcount_b200 import synth_cb as sc
from bam_readcount_b200.engine import Engine, load_library
spec = sc.Spec(seed=99, contig_len=1280 * 160, n_contigs=2)
L = spec.contig_len
jobs = [(0, dict(insertion_centric=True)), (1, dict(min_mapq=20, min_bq=20))]
batches = [spec.window_host(c, 0, 160)[0] for c, _ in jobs]
refs = [spec.ref_host(c, 0, L) for c, _ in jobs]
load_library()

def run(i, out, barrier=None):
    c, flags = jobs[i]
    try:
        e = Engine(**flags)
        try:
            if barrier is not None:
                barrier.wait(timeout=120)       # from here on both threads make their first use of the device's tables
            e.set_reference(c, f"chr{c + 1}", L, refs[i], 0)
            e.begin_region(c, 0, L, False)
            e.push_reads(batches[i])
            e.end_region()
            e.compute()
            pk = e.packed()
            out[i] = (pk.words.copy(), pk.sec.copy())
        finally:
            e.close()
    except BaseException as ex:
        out[i] = ex

both = [None, None]
barrier = threading.Barrier(2)
ths = [threading.Thread(target=run, args=(i, both, barrier)) for i in range(2)]
for t in ths:
    t.start()
for t in ths:
    t.join(timeout=300)
assert not any(t.is_alive() for t in ths), "a thread did not finish"
alone = [None, None]
for i in range(2):
    run(i, alone)
for x in both + alone:
    if isinstance(x, BaseException):
        raise x
np.savez(sys.argv[1], **{f"{tag}{i}_{k}": v for tag, res in (("both", both), ("alone", alone)) for i in range(2)
                         for k, v in zip(("words", "sec"), res[i])})
"""


@pytest.mark.gpu
def test_first_use_from_two_threads_in_a_fresh_process(tmp_path):
    """A fresh process whose two threads create a handle each and run their first pileup at the same time (the first runs
    upload the constant table, build the quotient tables and set the kernels' shared-memory limits): both give the records the
    same windows give run one after the other.  Run once, in a subprocess joined with a timeout."""
    out = str(tmp_path / "first_use.npz")
    p = subprocess.run([sys.executable, "-c", FIRST_USE, out], cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=600)
    assert p.returncode == 0, p.stdout[-4000:]
    with np.load(out) as z:
        for i in range(2):
            got = (z[f"both{i}_words"], z[f"both{i}_sec"])
            want = (z[f"alone{i}_words"], z[f"alone{i}_sec"])
            assert got[0].size > 0
            d = ic.diff_packed(f"thread {i} (contig {i})", got, want, 0)
            assert not d, d
