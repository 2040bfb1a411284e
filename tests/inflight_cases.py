"""Cases and helpers of tests/test_inflight_windows.py: the records bench.py's timed loops compute with every engine handle in
flight, taken from those loops as they run.

  * ``deal``: the C4 loop's round-robin schedule of windows over runners, and ``contig_changes_in_flight``: the windows at which
    a runner moves to a contig while another runner still holds the one it left;
  * ``Capture``: per-window copies of a handle's packed records, taken on a stream of their own in the order bench.py's
    gather_round takes them (wait for the window's kernels, copy, release the handle);
  * ``results_from_packed``: the full-width Results view of captured packed words and pool records (numpy restatement of the
    engine's ensure_wide), so a capture can be dumped and compared with the oracle;
  * ``check_window_against_oracle``: bench.py's oracle_dump recipe restated, run in worker processes (the Python dump of a
    window takes seconds).
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np

from bam_readcount_b200 import stream as st
from bam_readcount_b200 import synth_cb as sc
from bam_readcount_b200.engine import N_STATS, N_WORDS, SEC_RECORD_BYTES, PackedResults, Results

LIBS = [f"lib{i}" for i in range(8)]
KIND_WIDE = 8                    # pool records of kind >= 8 hold a whole site that escaped the packed word

# C4 at a small geometry: 3 contigs of 6 windows of 100 generator blocks
SMALL_SPEC = dict(seed=2024, contig_len=600 * sc.BLOCK_BP, n_contigs=3)
SMALL_WINDOWS_PER_CONTIG = 6
# C4 at its real geometry (bench.py CONFIGS["c4"]): 12.5 Mb windows, 10 per 125 Mb contig, on 2 contigs
REAL_SPEC = dict(seed=1234, contig_len=97656 * sc.BLOCK_BP, n_contigs=2)
REAL_WINDOWS_PER_CONTIG = 10
N_RUNNERS = 3
# A spin kernel of one thread at the head of a stream, ~25 ms on an H100: the kernels of a small window take less time than the
# host takes to enqueue it, so without one the GPU would run every window before the host queues the next (at the real C4
# geometry it is behind on its own)
GATE_CYCLES = 50_000_000


def hold(stream):
    """Hold `stream` back by GATE_CYCLES: what the host queues on it next runs after the host has moved on."""
    import torch
    with torch.cuda.stream(stream):
        torch.cuda._sleep(GATE_CYCLES)


def deal(n_windows: int, n_runners: int = N_RUNNERS) -> List[int]:
    """The runner of each window: bench.py's one_pass hands window k to runner k % n_runners."""
    return [k % n_runners for k in range(n_windows)]


def contig_changes_in_flight(windows: Sequence[st.Window], runners: Sequence[int], passes: int = 1) -> List[int]:
    """Indices (over `passes` passes) of the windows at which a runner leaves contig c for another while a second runner still
    holds c: the contig that is dropped only when its last holder moves on, while the new one is generated."""
    cur = {}
    out = []
    for k in range(passes * len(windows)):
        w, r = windows[k % len(windows)], runners[k % len(windows)]
        old = cur.get(r, -1)
        if old != -1 and old != w.contig and any(c == old for q, c in cur.items() if q != r):
            out.append(k)
        cur[r] = w.contig
    return out


def window_geometry(eng_rows: int, w: st.Window):
    """(words bytes, pool capacity in records) a handle holds for window w: the engine's default pool capacity."""
    rs = eng_rows * w.n_slots
    return rs * 4 * N_WORDS, max(rs // 4 + 4096, 1024)


class Capture:
    """Per-window copies of what a handle's window left in it, taken on a stream of their own: the stream waits for the
    window's `done` event, copies the packed words (or their checksum and a slot range of them), the whole pool and its
    record count into buffers of that window, then records `sent`, the event the runner waits for before it re-plans the
    handle.  Nothing waits on the host.  Buffers are allocated up front, so the loop allocates nothing."""

    def __init__(self, device, sizes, ranges=None):
        """sizes[k] = (words bytes, pool records) of window k; ranges[k] = (s0, s1, n_rows, n_slots): keep only slots
        [s0, s1) of the words, and a checksum of all of them."""
        import torch
        self.device = device
        self.stream = torch.cuda.Stream(device=device)
        self.ranges = ranges
        self.words, self.sec = [], []
        for k, (wb, cap) in enumerate(sizes):
            if ranges is None:
                self.words.append(torch.empty(wb, dtype=torch.uint8, device=device))
            else:
                s0, s1, rows, _ = ranges[k]
                self.words.append(torch.empty((N_WORDS, rows, s1 - s0), dtype=torch.int32, device=device))
            self.sec.append(torch.empty(cap * SEC_RECORD_BYTES, dtype=torch.uint8, device=device))
        self.count = torch.zeros(len(sizes), dtype=torch.int32, device=device)
        self.checksum = torch.zeros(len(sizes), dtype=torch.int64, device=device)

    def take(self, k: int, eng, done, sent):
        import torch
        s = self.stream
        with torch.cuda.stream(s):
            s.wait_event(done)                             # stream order only: the host does not wait for the window
            pk = eng.device_packed()
            rs = int(pk.n_rows) * int(pk.n_slots)
            words = st.alias_device_bytes(pk.words, rs * 4 * N_WORDS, self.device)
            sec = st.alias_device_bytes(pk.sec, int(pk.n_sec) * SEC_RECORD_BYTES, self.device)
            cnt = st.alias_device_bytes(pk.sec_count, 4, self.device).view(torch.int32)
            assert sec.numel() == self.sec[k].numel(), (k, sec.numel(), self.sec[k].numel())
            if self.ranges is None:
                assert words.numel() == self.words[k].numel(), (k, words.numel(), self.words[k].numel())
                self.words[k].copy_(words, non_blocking=True)
            else:
                s0, s1, rows, n_slots = self.ranges[k]
                assert rs == rows * n_slots, (k, rs, rows, n_slots)
                sc.checksum_device(words, self.checksum[k:k + 1], s.cuda_stream)
                self.words[k].copy_(words.view(torch.int32).view(N_WORDS, rows, n_slots)[:, :, s0:s1], non_blocking=True)
            self.sec[k].copy_(sec, non_blocking=True)
            self.count[k:k + 1].copy_(cnt, non_blocking=True)
            sent.record(s)                                 # the records have left the handle: it may be re-planned

    def host(self, k: int, n_rows: int, what: str = ""):
        """(words uint32 [N_WORDS, rows, slots], pool records uint32 [count, 18]) of window k (call after a synchronize)."""
        n = int(self.count[k].item())
        cap = self.sec[k].numel() // SEC_RECORD_BYTES
        assert 0 <= n <= cap, f"{what or f'window {k}'}: pool count {n} outside the pool's {cap} records"
        w = self.words[k].cpu().numpy().view(np.uint32)
        w = w.reshape(N_WORDS, n_rows, -1)
        sec = self.sec[k][:n * SEC_RECORD_BYTES].cpu().numpy().view(np.uint32).reshape(n, SEC_RECORD_BYTES // 4)
        return w, sec


def sorted_records(sec: np.ndarray) -> np.ndarray:
    """Pool records without their chain link (column 1), sorted: pool order depends on thread timing."""
    r = np.delete(sec, 1, axis=1)
    return r[np.lexsort(r.T[::-1])] if len(r) else r


def record_digest(sec: np.ndarray) -> np.ndarray:
    """An order-independent digest of pool records: a 64-bit hash of every record without its chain link, sorted."""
    r = np.delete(sec, 1, axis=1).astype(np.uint64)
    h = np.full(len(r), 0xCBF29CE484222325, dtype=np.uint64)
    with np.errstate(over="ignore"):
        for c in range(r.shape[1]):
            h = (h ^ r[:, c]) * np.uint64(0x100000001B3)
            h ^= h >> np.uint64(31)
    return np.sort(h)


def site_of(slot: int, n_slots: int, first_pos: int) -> str:
    row, s = divmod(int(slot), n_slots)
    return f"row {row}, site {first_pos + s} (0-based)"


def diff_packed(what: str, got, want, first_pos: int) -> Optional[str]:
    """None when two (words, pool records) pairs are the same records; else where they first differ."""
    gw, gs = got
    ww, ws = want
    if gw.shape != ww.shape:
        return f"{what}: words shape {gw.shape} != {ww.shape}"
    bad = np.argwhere(gw != ww)
    if len(bad):
        wd, row, s = (int(x) for x in bad[0])
        return f"{what}: {len(bad)} packed words differ, first word {wd} of row {row}, site {first_pos + s} (0-based)"
    if len(gs) != len(ws):
        return f"{what}: {len(gs)} pool records, want {len(ws)}"
    a, b = sorted_records(gs), sorted_records(ws)
    bad = np.nonzero((a != b).any(axis=1))[0]
    if len(bad):
        j = int(bad[0])
        return (f"{what}: {len(bad)} sorted pool records differ, first at {site_of(min(a[j, 0], b[j, 0]), gw.shape[2], first_pos)}: "
                f"{a[j].tolist()} != {b[j].tolist()}")
    return None


def results_from_packed(words: np.ndarray, sec: np.ndarray, regions: List[dict]) -> Results:
    """The full-width view of packed words [N_WORDS, rows, slots] and pool records, as brc_get_results gives it: escaped
    sites filled from their record, keys chained per (row, slot) (chain order is immaterial to the dump)."""
    n_rows, n_slots = int(words.shape[1]), int(words.shape[2])
    pk = PackedResults.__new__(PackedResults)
    pk.n_rows, pk.n_slots, pk.words, pk.n_sec, pk.sec = n_rows, n_slots, words, len(sec), sec
    ncover, npass, flags, pbase, ps = pk.widen()
    r = Results.__new__(Results)
    r.n_rows, r.n_slots, r.regions = n_rows, n_slots, [dict(g) for g in regions]
    r.ncover, r.npass, r.flags, r.pbase, r.pstats = ncover, npass, flags, pbase, ps
    ns = len(sec)
    kind = (sec[:, 2] & 0xFF).astype(np.uint8) if ns else np.zeros(0, np.uint8)
    r.n_sec = ns
    r.sec_kind = np.where(kind >= KIND_WIDE, 0xFF, kind).astype(np.uint8)
    r.sec_len = (sec[:, 2] >> 8).astype(np.int32) if ns else np.zeros(0, np.int32)
    r.sec_read = sec[:, 3].view(np.int32).astype(np.int64) if ns else np.zeros(0, np.int64)
    r.sec_qpos = sec[:, 4].view(np.int32).copy() if ns else np.zeros(0, np.int32)
    r.sec_stats = sec[:, 5:5 + N_STATS].T.copy() if ns else np.zeros((N_STATS, 0), np.uint32)
    head = np.full(n_rows * n_slots, -1, dtype=np.int32)
    nxt = np.full(ns, -1, dtype=np.int32)
    keys = np.nonzero(kind < KIND_WIDE)[0]
    if len(keys):
        slot = sec[keys, 0].astype(np.int64)
        order = keys[np.argsort(slot, kind="stable")]
        ss = sec[order, 0].astype(np.int64)
        same = ss[1:] == ss[:-1]
        nxt[order[:-1][same]] = order[1:][same]
        first = np.concatenate([[True], ~same])
        head[ss[first]] = order[first]
    r.sec_head = head.reshape(n_rows, n_slots)
    r.sec_next = nxt
    return r


def slot_range(words: np.ndarray, sec: np.ndarray, s0: int, s1: int, n_slots: int):
    """The pool records of slots [s0, s1) of every row, re-addressed to a view that holds only those slots."""
    slot = sec[:, 0].astype(np.int64)
    row, s = slot // n_slots, slot % n_slots
    keep = (s >= s0) & (s < s1)
    out = sec[keep].copy()
    out[:, 0] = (row[keep] * (s1 - s0) + s[keep] - s0).astype(np.uint32)
    return out


def oracle_dump(spec, flags, contig, pos_lo, pos_hi, lib_names):
    """bench.py's oracle_dump: the CPU oracle on the host-generated reads around [pos_lo, pos_hi), region (pos_lo+1, pos_hi)
    with halo pos_lo.  Returns (dump text, host batch, its first block, (reference window start, reference bytes))."""
    from oracle.oracle import Oracle
    blo = max(pos_lo // sc.BLOCK_BP - 1, 0)
    bhi = min(-(-pos_hi // sc.BLOCK_BP), spec.blocks_per_contig())
    hb, _ = spec.window_host(contig, blo, bhi)
    beg, end = pos_lo + 1, pos_hi
    ref_end = min(spec.contig_len, bhi * sc.BLOCK_BP + 400)
    ref = spec.ref_host(contig, 0, ref_end) if ref_end < 50_000_000 else None
    wb = 0
    if ref is None:
        wb = max(blo * sc.BLOCK_BP - 400, 0)
        ref = spec.ref_host(contig, wb, ref_end - wb)
    o = Oracle(lib_names=lib_names, **flags)
    sub = hb.select(hb.fetch(contig, beg - 1, end))
    o.region(sub, tid=contig, beg=beg, end=end, contig=f"chr{contig + 1}", chrom_len=spec.contig_len, ref_seq=ref, ref_win_beg=wb,
             site_list_mode=False)
    return o.dump(), hb, blo, (wb, ref)


def check_window_against_oracle(label: str, spec_kw: dict, flags: dict, lib_names, contig: int, pos_lo: int, pos_hi: int,
                                blk_lo: int, res: Results) -> Optional[str]:
    """None when the dump of sites [pos_lo, pos_hi) of `res` (region 0; its reads start at block blk_lo) is the oracle's."""
    from cases import first_diff
    od, hb, blo, (wb, ref) = oracle_dump(sc.Spec(**spec_kw), flags, contig, pos_lo, pos_hi, lib_names)
    ed = res.dump_range(hb, {contig: (wb, ref)}, 0, pos_lo, pos_hi, read_offset=(blo - blk_lo) * sc.BLOCK_READS)
    if not od:
        return f"{label}: the oracle printed nothing for sites [{pos_lo}, {pos_hi})"
    return None if ed == od else f"{label}: " + first_diff(ed, od)
