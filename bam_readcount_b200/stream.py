"""Streaming / sharded driver of the device-resident path (SURVEY.md §8e; R:src/exe/bam-readcount/bamreadcount.cpp:574-608, 641-657).

The reference's unit of independence is the region: a fresh pileup buffer per region (R:…:591, :650), the deletion queue
cleared per site-list line (R:…:605).  A genome is therefore cut into WINDOWS (regions of a few Mb — what fits HBM next to its
results), windows are dealt to ranks as contiguous SHARDS balanced by a coverage weight (the BAI linear index for a real BAM,
uniform for the synthetic genome), and every rank walks its shard on three engine handles: while window w runs on one handle's
stream, the next windows' reads are produced (generator / already resident in HBM) and planned on the others.  Window [b, e) computes
site b-1 as its halo (R:…:269 vs :414), so no state crosses a window or a rank.

The only inter-rank traffic is the ORDERED EMIT: every rank sends the packed records of each finished window to rank 0
(`GatherRing`: ncclSend/ncclRecv through torch.distributed P2P ops inside one group per round; `round_fixed` sends
messages whose sizes follow from the shard plan, queued behind the kernels with no host synchronisation; `round` is the
variable-size form with an all-gather of the byte counts first); ranks hold ascending site ranges, so rank 0 spools shard by
shard in rank order, into two spool sets per source, and consumes them on an emitter stream of its own.
"""
from __future__ import annotations

import ctypes as C
import weakref
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import synth_cb
from .engine import CRegion, Engine, N_WORDS, SEC_RECORD_BYTES


@dataclass(frozen=True)
class Window:
    contig: int
    blk_lo: int        # generator blocks whose reads are needed: [blk_lo, blk_hi)
    blk_hi: int
    beg: int           # sites [beg, end) are this window's output (0-based, end exclusive); site beg-1 is the halo
    end: int

    @property
    def first_pos(self) -> int:
        return max(self.beg - 1, 0)

    @property
    def n_slots(self) -> int:
        return self.end - self.first_pos

    @property
    def n_sites(self) -> int:
        return self.end - self.beg


def wgs_windows(spec: synth_cb.Spec, windows_per_contig: int) -> List[Window]:
    """All windows of the synthetic genome in genome order.  A window's reads are the blocks that can overlap
    [beg-1, end): its own blocks plus the one before (a read spans at most 153 bp < one block)."""
    nb = spec.blocks_per_contig()
    per = -(-nb // windows_per_contig)
    out = []
    for c in range(spec.n_contigs):
        for lo in range(0, nb, per):
            hi = min(nb, lo + per)
            out.append(Window(c, max(lo - 1, 0), hi, lo * synth_cb.BLOCK_BP, hi * synth_cb.BLOCK_BP))
    return out


def plan_shards_weighted(weights: Sequence[float], world_size: int) -> List[Tuple[int, int]]:
    """Contiguous partition of units 0..n-1 into `world_size` shards of about equal total weight (the coverage
    proxy: BAI linear-index byte deltas for a BAM, read counts for a generated genome).  Returns [lo, hi) per rank;
    every unit belongs to exactly one shard, shards are ascending, some may be empty when n < world_size."""
    w = np.asarray(weights, dtype=np.float64)
    n = int(w.shape[0])
    assert world_size >= 1
    tot = float(w.sum())
    if n == 0:
        return [(0, 0)] * world_size
    if tot <= 0:
        w = np.ones(n)
        tot = float(n)
    cum = np.concatenate([[0.0], np.cumsum(w)])
    cuts = [0]
    for r in range(1, world_size):
        target = tot * r / world_size
        c = int(np.searchsorted(cum, target, side="left"))
        # the cut that leaves the prefix closest to the target
        if c > 0 and abs(cum[c - 1] - target) <= abs(cum[min(c, n)] - target):
            c -= 1
        c = min(max(c, cuts[-1]), n)
        cuts.append(c)
    cuts.append(n)
    return [(cuts[i], cuts[i + 1]) for i in range(world_size)]


def window_region(w: Window) -> CRegion:
    return CRegion(w.contig, w.beg, w.end, 0, 0, 0, 0, w.first_pos, w.n_slots)


class _CudaView:
    """Wraps a raw device pointer so torch.as_tensor can alias it (no copy): the engine owns the memory."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1", "data": (int(ptr), False), "version": 2}


def alias_device_bytes(ptr: int, nbytes: int, device):
    import torch
    if nbytes == 0:
        return torch.empty(0, dtype=torch.uint8, device=device)
    return torch.as_tensor(_CudaView(ptr, nbytes), device=device)


def reference_length(spec: synth_cb.Spec) -> int:
    return spec.contig_len if spec.mode == synth_cb.WGS else spec.deep_contig_len()


class DeviceReference:
    """One contig's reference characters in HBM, generated on one stream; every stream that reads them waits for that first."""

    def __init__(self, spec: synth_cb.Spec, contig: int, stream, device):
        import torch
        self.length = reference_length(spec)
        with torch.cuda.stream(stream):
            self.ascii = torch.empty(self.length + 64, dtype=torch.uint8, device=device)
        rc = synth_cb.load().brc_synth_ref_device(C.byref(spec.c), contig, 0, self.length, self.ascii.data_ptr(), stream.cuda_stream)
        assert rc == 0, rc
        self.ready = torch.cuda.Event()
        self.ready.record(stream)

    def use_on(self, stream):
        stream.wait_event(self.ready)
        self.ascii.record_stream(stream)          # the allocator must not hand the bytes out again before this stream has read them


class ContigReferences:
    """The reference characters of the contigs that the runners of one generated genome on one device are on.  A contig is
    generated once, on the stream of the first runner that moves to it, and dropped when the last runner holding it moves on
    or is closed.  Runners deal a contig's windows round-robin, so without sharing every runner would generate every contig
    again.  Holders are held weakly: a runner dropped without close() stops holding its contig, which goes at the next move."""

    def __init__(self):
        self._live = {}            # contig -> (reference, WeakSet of the runners holding it)
        self.generated = 0

    def move(self, runner, old: int, new: int):
        """`runner` leaves contig `old` for `new`; returns `new`'s reference, ready to be read on `runner.stream`."""
        self.release(runner, old)
        for c in [c for c, (_, holders) in self._live.items() if not holders and c != new]:
            del self._live[c]
        entry = self._live.get(new)
        if entry is None:
            entry = self._live[new] = (runner.generate_reference(new), weakref.WeakSet())
            self.generated += 1
        entry[0].use_on(runner.stream)
        entry[1].add(runner)
        return entry[0]

    def release(self, runner, contig: int):
        entry = self._live.get(contig)
        if entry is not None:
            entry[1].discard(runner)
            if not entry[1]:
                del self._live[contig]

    def live(self) -> List[int]:
        return sorted(c for c, (_, holders) in self._live.items() if holders)


_shared_references = weakref.WeakKeyDictionary()      # spec -> {device index: ContigReferences}


def shared_references(spec: synth_cb.Spec, device_index: int) -> ContigReferences:
    """The ContigReferences every WindowRunner of `spec` on that device uses."""
    return _shared_references.setdefault(spec, {}).setdefault(device_index, ContigReferences())


class WindowRunner:
    """One engine handle + its generator buffers: runs one window at a time on its own stream.  The runners of one spec on one
    device share the reference characters of their contigs (ContigReferences); each handle encodes them into its own window."""

    def __init__(self, spec: synth_cb.Spec, max_window_reads: int, device, flags: dict, lib_names: Sequence[str] = ()):
        import torch
        self.spec, self.device = spec, device
        index = device.index if hasattr(device, "index") and device.index is not None else 0
        self.eng = Engine(device=index, lib_names=lib_names, **flags)
        self.dw = synth_cb.DeviceWindow(spec, max_window_reads, device)
        self.stream = torch.cuda.Stream(device=device)
        self.done = torch.cuda.Event()            # kernels of the current window finished
        self.sent = torch.cuda.Event()            # its records left the handle (gather) — safe to re-plan
        self.refs = shared_references(spec, index)
        self.cur_contig = -1
        self.window: Optional[Window] = None
        self.n_sec_host = None                    # pinned int32[1]: the window's record count
        self.busy = False

    def close(self):
        self.refs.release(self, self.cur_contig)
        self.eng.close()

    def generate_reference(self, contig: int) -> DeviceReference:
        return DeviceReference(self.spec, contig, self.stream, self.device)

    def _ensure_reference(self, contig: int):
        if contig == self.cur_contig:
            return
        ref = self.refs.move(self, self.cur_contig, contig)
        self.eng.set_reference_device(contig, f"chr{contig + 1}", ref.length, 0, ref.ascii.data_ptr(), ref.length, self.stream.cuda_stream)
        self.cur_contig = contig

    def launch(self, w: Window, sec_cap: int = 0, resident=None):
        """Enqueue the engine's kernels for window w; its reads are generated in HBM first, unless `resident` (a DeviceWindow
        that already holds them) is given.  Returns immediately."""
        import torch
        if self.busy:
            self.done.synchronize()
            self.sent.synchronize()
        sp = self.stream.cuda_stream
        self._ensure_reference(w.contig)
        dw = resident if resident is not None else self.dw
        n = dw.n_reads if resident is not None else dw.fill(w.contig, w.blk_lo, w.blk_hi, sp)
        reg = window_region(w)
        reg.read_hi = n
        self.eng.plan_device([reg], n, sec_cap)
        self.eng.run_device(dw.c_batch(), None, sp)
        if self.n_sec_host is None:
            self.n_sec_host = torch.zeros(1, dtype=torch.int32).pin_memory()
        pk = self.eng.device_packed()
        with torch.cuda.stream(self.stream):
            cnt = alias_device_bytes(pk.sec_count, 4, self.device).view(torch.int32)
            self.n_sec_host.copy_(cnt, non_blocking=True)
            self.done.record(self.stream)
            self.sent.record(self.stream)
        self.window, self.busy = w, True

    def packed_tensors_fixed(self, sec_cap_records: int):
        """(words, sec[:cap], count) aliasing the engine's device records WITHOUT waiting for the window: every size is known from
        the window's geometry, so a gather can be queued behind the kernels (stream order) with no host synchronisation."""
        pk = self.eng.device_packed()
        rs = int(pk.n_rows) * int(pk.n_slots)
        cap = min(int(sec_cap_records), int(pk.n_sec))
        return (alias_device_bytes(pk.words, rs * 4 * N_WORDS, self.device), alias_device_bytes(pk.sec, cap * SEC_RECORD_BYTES, self.device),
                alias_device_bytes(pk.sec_count, 4, self.device))

    def packed_tensors(self):
        """(words bytes, sec bytes) aliasing the engine's device records of the finished window (call after done)."""
        pk = self.eng.device_packed()
        rs = int(pk.n_rows) * int(pk.n_slots)
        n_sec = int(self.n_sec_host[0])
        if n_sec > int(pk.n_sec):
            raise RuntimeError(f"secondary pool overflow: {n_sec} records > capacity {int(pk.n_sec)} (raise sec_cap)")
        return (alias_device_bytes(pk.words, rs * 4 * N_WORDS, self.device), alias_device_bytes(pk.sec, n_sec * SEC_RECORD_BYTES, self.device))


class GatherRing:
    """Ordered-emit transport: rank 0 receives every other rank's packed window records over the process group.

    One ROUND = the k-th window of every rank: ONE group of point-to-point ops (NCCL: ncclGroupStart / ncclSend / ncclRecv /
    ncclGroupEnd) — the sends of every rank > 0, the matching receives on rank 0 into that round's per-source spool buffers (two
    sets, alternating).  `round_fixed`: message sizes known from the shard plan (words, a bounded pool message, the 4-byte true
    count), nothing waits on the host.  `round`: an all-gather of (words bytes, pool bytes) first, then exact sizes.
    `consume(src, words, sec)` is called on rank 0 for every received pair on the emitter stream (bench.py checksums the bytes)."""

    def __init__(self, rank: int, world: int, device, max_words_bytes: int, max_sec_bytes: int, group=None, consume=None):
        import torch
        self.rank, self.world, self.device, self.group, self.consume = rank, world, device, group, consume
        self.sizes = torch.zeros(2, dtype=torch.int64, device=device)
        self.all_sizes = torch.zeros(2 * world, dtype=torch.int64, device=device)
        # rank 0: TWO spool sets per source, alternating by round, and a stream of its own for the emitter: the receives of
        # round k+1 land while round k is still being consumed, so the NVLink ingress never idles behind the consumer
        self.spool_w, self.spool_s = {}, {}
        self.emit_stream = None
        self.arrived, self.consumed = [], []
        if rank == 0 and world > 1:
            for src in range(1, world):
                self.spool_w[src] = [torch.empty(max_words_bytes, dtype=torch.uint8, device=device) for _ in range(2)]
                self.spool_s[src] = [torch.empty(max_sec_bytes, dtype=torch.uint8, device=device) for _ in range(2)]
            if torch.device(device).type == "cuda":     # (the gloo tests run the same protocol on CPU tensors: consumed inline)
                self.emit_stream = torch.cuda.Stream(device=device)
                self.arrived = [torch.cuda.Event() for _ in range(2)]
                self.consumed = [torch.cuda.Event() for _ in range(2)]
                for ev in self.consumed:
                    ev.record()
        self.bytes_received = 0
        self.rounds = 0

    @staticmethod
    def spool_bytes(world: int, max_words_bytes: int, max_sec_bytes: int) -> int:
        """HBM rank 0 sets aside for the spools."""
        return 2 * (world - 1) * (max_words_bytes + max_sec_bytes) if world > 1 else 0

    def join(self, stream):
        """Make `stream` wait for the emitter (rank 0)."""
        if self.emit_stream is not None:
            stream.wait_stream(self.emit_stream)

    def _consume_round(self, got, p):
        import torch
        if self.consume is None or not got:
            return
        if self.emit_stream is None:
            for src, tw, ts in got:
                self.consume(src, tw, ts)
            return
        cur = torch.cuda.current_stream()
        self.arrived[p].record(cur)
        self.emit_stream.wait_event(self.arrived[p])
        with torch.cuda.stream(self.emit_stream):
            for src, tw, ts in got:
                self.consume(src, tw, ts)
            self.consumed[p].record(self.emit_stream)

    def round_fixed(self, mine, peers):
        """Size-exchange-free round: `mine` = (words, sec[:cap], count4) uint8 device tensors of this rank's window or None;
        `peers` (rank 0 only) = {src: (words_bytes, sec_bytes)} of what each peer sends this round (known from the shard plan).
        Nothing here waits on the host: the ops are queued on the current stream behind the kernels that produce the data."""
        import torch.distributed as dist
        if self.world == 1:
            return
        import torch
        ops, got = [], []
        p = self.rounds & 1
        if self.rank == 0:
            if self.emit_stream is not None:
                torch.cuda.current_stream().wait_event(self.consumed[p])      # the emitter is done with this spool set
            for src, (nw, ns) in sorted(peers.items()):
                sw, ss = self.spool_w[src][p], self.spool_s[src][p]
                if nw > sw.numel() or ns + 4 > ss.numel():
                    raise RuntimeError(f"gather spool too small for rank {src}: {nw}/{ns} bytes")
                tw, ts, tc = sw[:nw], ss[:ns], ss[ns:ns + 4]
                ops += [dist.P2POp(dist.irecv, tw, src, group=self.group), dist.P2POp(dist.irecv, ts, src, group=self.group),
                        dist.P2POp(dist.irecv, tc, src, group=self.group)]
                got.append((src, tw, ts))
                self.bytes_received += nw + ns + 4
        elif mine is not None:
            ops = [dist.P2POp(dist.isend, t, 0, group=self.group) for t in mine]
        if ops:
            for req in dist.batch_isend_irecv(ops):
                req.wait()
        if self.rank == 0:
            self._consume_round(got, p)
        self.rounds += 1

    def round(self, words, sec):
        """words / sec: uint8 device tensors of this rank's finished window (empty tensors when it has none this round).
        Collective: every rank calls it once per round, on the stream the tensors are ready on."""
        import torch
        import torch.distributed as dist
        if self.world == 1:
            return
        self.sizes[0] = int(words.numel())
        self.sizes[1] = int(sec.numel())
        dist.all_gather_into_tensor(self.all_sizes, self.sizes, group=self.group)
        sz = self.all_sizes.cpu().tolist()
        ops, got = [], []
        p = self.rounds & 1
        if self.rank == 0:
            if self.emit_stream is not None:
                torch.cuda.current_stream().wait_event(self.consumed[p])
            for src in range(1, self.world):
                nw, ns = int(sz[2 * src]), int(sz[2 * src + 1])
                sw, ss = self.spool_w[src][p], self.spool_s[src][p]
                if nw > sw.numel() or ns > ss.numel():
                    raise RuntimeError(f"gather spool too small for rank {src}: {nw}/{ns} bytes")
                tw, ts = sw[:nw], ss[:ns]
                if nw:
                    ops.append(dist.P2POp(dist.irecv, tw, src, group=self.group))
                if ns:
                    ops.append(dist.P2POp(dist.irecv, ts, src, group=self.group))
                got.append((src, tw, ts))
                self.bytes_received += nw + ns
        else:
            if words.numel():
                ops.append(dist.P2POp(dist.isend, words, 0, group=self.group))
            if sec.numel():
                ops.append(dist.P2POp(dist.isend, sec, 0, group=self.group))
        if ops:
            for req in dist.batch_isend_irecv(ops):
                req.wait()
        if self.rank == 0:
            self._consume_round(got, p)
        self.rounds += 1
