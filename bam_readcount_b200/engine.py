"""ctypes binding of libbrc_engine.so (include/brc_engine.h) — the Python host of the engine.

The host mirrors the reference's region driver: ``Engine.begin_region / push_reads /
end_region`` are ``bam_plbuf_init / fetch_func+bam_plbuf_push / bam_plbuf_push(0)``
(R:src/exe/bam-readcount/bamreadcount.cpp:588-605).  There is NO CPU fallback: if the CUDA
library is missing or no device is usable, construction raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence

import numpy as np

from .batch import ReadBatch

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libbrc_engine.so")
if os.environ.get("BRC_ENGINE_LIB"):        # debug hook: an instrumented build of the same library
    LIB_PATH = os.environ["BRC_ENGINE_LIB"]

N_STATS = 13
KIND_INS, KIND_DEL, NO_BASE = 6, 7, 255
NT = "=ACGTN"
_CANON = np.array([0, 1, 2, 5, 3, 5, 5, 5, 4, 5, 5, 5, 5, 5, 5, 5], dtype=np.uint8)
_FLOAT_STATS = (6, 7, 10, 12)


class BrcError(RuntimeError):
    def __init__(self, status: int, msg: str):
        super().__init__(f"brc status {status}: {msg}")
        self.status = status


class Config(C.Structure):
    _fields_ = [("min_mapq", C.c_int32), ("min_bq", C.c_int32), ("max_cnt", C.c_int32), ("per_lib", C.c_int32),
                ("insertion_centric", C.c_int32), ("n_libs", C.c_int32), ("device", C.c_int32), ("reserved", C.c_int32)]


class CReadBatch(C.Structure):
    _fields_ = [("n_reads", C.c_int64), ("tid", C.c_void_p), ("pos", C.c_void_p), ("flag", C.c_void_p),
                ("mapq", C.c_void_p), ("lib", C.c_void_p), ("l_qseq", C.c_void_p), ("nm", C.c_void_p),
                ("sm", C.c_void_p), ("cigar_off", C.c_void_p), ("cigar", C.c_void_p), ("seq_off", C.c_void_p),
                ("seq", C.c_void_p), ("qual_off", C.c_void_p), ("qual", C.c_void_p)]


class CRegion(C.Structure):
    _fields_ = [("tid", C.c_int32), ("beg", C.c_int32), ("end", C.c_int32), ("site_list_mode", C.c_int32),
                ("read_lo", C.c_int64), ("read_hi", C.c_int64), ("slot_base", C.c_int64), ("first_pos", C.c_int32),
                ("n_slots", C.c_int32)]


class CResults(C.Structure):
    _fields_ = [("n_regions", C.c_int64), ("regions", C.POINTER(CRegion)), ("n_rows", C.c_int32), ("n_slots", C.c_int64),
                ("ncover", C.c_void_p), ("npass", C.c_void_p), ("flags", C.c_void_p), ("pbase", C.c_void_p),
                ("sec_head", C.c_void_p), ("pstats", C.c_void_p), ("n_sec", C.c_int64), ("sec_next", C.c_void_p),
                ("sec_kind", C.c_void_p), ("sec_len", C.c_void_p), ("sec_read", C.c_void_p), ("sec_qpos", C.c_void_p),
                ("sec_stats", C.c_void_p)]


class CBamSpan(C.Structure):
    _fields_ = [("comp", C.c_void_p), ("comp_len", C.c_int64), ("n_entry", C.c_int64), ("entry", C.c_void_p), ("end_voff", C.c_int64),
                ("tid", C.c_int32), ("n_rg", C.c_int32), ("rg_id", C.c_void_p), ("rg_lib", C.c_void_p)]


class CSecRecord(C.Structure):
    _fields_ = [("slot", C.c_uint32), ("next", C.c_int32), ("kind_len", C.c_uint32), ("read", C.c_int32), ("qpos", C.c_int32),
                ("stats", C.c_uint32 * 13)]


class CPackedResults(C.Structure):
    """brc_packed_results: the 32 B/site records the kernels write (include/brc_engine.h)."""
    _fields_ = [("n_regions", C.c_int64), ("regions", C.POINTER(CRegion)), ("n_rows", C.c_int32), ("n_slots", C.c_int64),
                ("words", C.c_void_p), ("n_sec", C.c_int64), ("sec", C.c_void_p), ("sec_count", C.c_void_p)]


class CSiteFilter(C.Structure):
    _fields_ = [("min_alt_count", C.c_int32), ("reserved", C.c_int32), ("min_alt_fraction", C.c_double)]


class CSelectedResults(C.Structure):
    """brc_selected_results: the sites a site filter shipped (include/brc_engine.h)."""
    _fields_ = [("n_regions", C.c_int64), ("regions", C.POINTER(CRegion)), ("n_rows", C.c_int32), ("n_slots", C.c_int64),
                ("n_sites", C.c_int64), ("site", C.c_void_p), ("emit", C.c_void_p), ("words", C.c_void_p), ("n_sec", C.c_int64),
                ("sec", C.c_void_p)]


N_WORDS = 8
SEC_RECORD_BYTES = 72

EXPORTS = [
    "brc_abi_version", "brc_create", "brc_destroy", "brc_last_error", "brc_strerror", "brc_set_reference", "brc_set_reference_device", "brc_reset",
    "brc_begin_region", "brc_push_read", "brc_push_reads", "brc_end_region", "brc_decode_bam_span", "brc_push_bam_span", "brc_fetch_decoded_batch", "brc_compute", "brc_get_results",
    "brc_get_warning_counts", "brc_format_text", "brc_format_window", "brc_write_text", "brc_set_queue_carry", "brc_plan_device", "brc_run_device", "brc_device_packed_results", "brc_get_packed_results",
    "brc_fetch_device_results", "brc_last_launch_count", "brc_last_h2d_bytes", "brc_host_alloc", "brc_host_free", "brc_last_stage_ms", "brc_selftest_fastmath",
    "brc_set_site_filter", "brc_get_selected_results",
]

_lib = None


def load_library(path: Optional[str] = None) -> C.CDLL:
    """Load the CUDA engine.  Fails loudly when it has not been built."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise RuntimeError(f"{p} is missing: build the CUDA extension first (python -m bam_readcount_b200.build); "
                           "there is no CPU fallback")
    lib = C.CDLL(p)
    lib.brc_create.argtypes = [C.POINTER(Config), C.POINTER(C.c_void_p)]
    lib.brc_destroy.argtypes = [C.c_void_p]
    lib.brc_destroy.restype = None
    lib.brc_last_error.argtypes = [C.c_void_p]
    lib.brc_last_error.restype = C.c_char_p
    lib.brc_strerror.argtypes = [C.c_int]
    lib.brc_strerror.restype = C.c_char_p
    lib.brc_set_reference.argtypes = [C.c_void_p, C.c_int32, C.c_char_p, C.c_int64, C.c_int64, C.c_char_p, C.c_int64]
    lib.brc_set_reference_device.argtypes = [C.c_void_p, C.c_int32, C.c_char_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
    lib.brc_reset.argtypes = [C.c_void_p]
    lib.brc_begin_region.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    lib.brc_push_read.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_uint16, C.c_uint8, C.c_uint16, C.c_int32,
                                  C.c_int32, C.c_int32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.brc_push_reads.argtypes = [C.c_void_p, C.POINTER(CReadBatch)]
    lib.brc_end_region.argtypes = [C.c_void_p]
    lib.brc_decode_bam_span.argtypes = [C.c_void_p, C.POINTER(CBamSpan), C.POINTER(CReadBatch), C.c_void_p]
    lib.brc_push_bam_span.argtypes = [C.c_void_p, C.POINTER(CBamSpan)]
    lib.brc_fetch_decoded_batch.argtypes = [C.c_void_p, C.POINTER(CReadBatch)]
    lib.brc_compute.argtypes = [C.c_void_p]
    lib.brc_get_results.argtypes = [C.c_void_p, C.POINTER(CResults)]
    lib.brc_get_warning_counts.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
    lib.brc_format_text.argtypes = [C.c_void_p, C.c_int64, C.POINTER(C.c_char_p), C.c_void_p, C.c_int64]
    lib.brc_format_text.restype = C.c_int64
    lib.brc_format_window.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.POINTER(C.c_char_p), C.c_void_p, C.c_int64]
    lib.brc_format_window.restype = C.c_int64
    lib.brc_write_text.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.POINTER(C.c_char_p), C.c_int]
    lib.brc_write_text.restype = C.c_int64
    lib.brc_set_queue_carry.argtypes = [C.c_void_p, C.c_int]
    lib.brc_plan_device.argtypes = [C.c_void_p, C.POINTER(CRegion), C.c_int64, C.c_int64, C.c_int64]
    lib.brc_run_device.argtypes = [C.c_void_p, C.POINTER(CReadBatch), C.c_void_p, C.c_void_p]
    lib.brc_device_packed_results.argtypes = [C.c_void_p, C.POINTER(CPackedResults)]
    lib.brc_get_packed_results.argtypes = [C.c_void_p, C.POINTER(CPackedResults)]
    lib.brc_fetch_device_results.argtypes = [C.c_void_p, C.c_void_p]
    lib.brc_selftest_fastmath.argtypes = [C.c_void_p, C.c_int32]
    lib.brc_selftest_fastmath.restype = C.c_int64
    lib.brc_last_launch_count.argtypes = [C.c_void_p]
    lib.brc_last_h2d_bytes.argtypes = [C.c_void_p]
    lib.brc_last_h2d_bytes.restype = C.c_int64
    lib.brc_last_stage_ms.argtypes = [C.c_void_p, C.c_int]
    lib.brc_last_stage_ms.restype = C.c_float
    lib.brc_set_site_filter.argtypes = [C.c_void_p, C.POINTER(CSiteFilter)]
    lib.brc_get_selected_results.argtypes = [C.c_void_p, C.POINTER(CSelectedResults)]
    if path is None:
        _lib = lib
    return lib


def _np_view(ptr, n, dtype):
    if n == 0 or not ptr:
        return np.zeros(0, dtype=dtype)
    buf = (C.c_char * (int(n) * np.dtype(dtype).itemsize)).from_address(ptr)
    return np.frombuffer(buf, dtype=dtype, count=int(n))


class Results:
    """Host copy (numpy) of one brc_compute's output."""

    def __init__(self, r: CResults):
        self.n_rows = int(r.n_rows)
        self.n_slots = int(r.n_slots)
        rs = self.n_rows * self.n_slots
        self.regions = [r.regions[i] for i in range(int(r.n_regions))]
        self.regions = [dict(tid=g.tid, beg=g.beg, end=g.end, site_list_mode=g.site_list_mode, read_lo=g.read_lo,
                             read_hi=g.read_hi, slot_base=g.slot_base, first_pos=g.first_pos, n_slots=g.n_slots)
                        for g in self.regions]
        self.ncover = _np_view(r.ncover, rs, np.uint32).reshape(self.n_rows, self.n_slots).copy()
        self.npass = _np_view(r.npass, rs, np.uint32).reshape(self.n_rows, self.n_slots).copy()
        self.flags = _np_view(r.flags, rs, np.uint8).reshape(self.n_rows, self.n_slots).copy()
        self.pbase = _np_view(r.pbase, rs, np.uint8).reshape(self.n_rows, self.n_slots).copy()
        self.sec_head = _np_view(r.sec_head, rs, np.int32).reshape(self.n_rows, self.n_slots).copy()
        self.pstats = _np_view(r.pstats, rs * N_STATS, np.uint32).reshape(N_STATS, self.n_rows, self.n_slots).copy()
        ns = int(r.n_sec)
        self.n_sec = ns
        self.sec_next = _np_view(r.sec_next, ns, np.int32).copy()
        self.sec_kind = _np_view(r.sec_kind, ns, np.uint8).copy()
        self.sec_len = _np_view(r.sec_len, ns, np.int32).copy()
        self.sec_read = _np_view(r.sec_read, ns, np.int64).copy()
        self.sec_qpos = _np_view(r.sec_qpos, ns, np.int32).copy()
        self.sec_stats = _np_view(r.sec_stats, ns * N_STATS, np.uint32).reshape(N_STATS, ns).copy()

    # ---- checker-facing view: same text as oracle/brc_oracle.c's raw dump -------------------
    def dump(self, pushed: ReadBatch, refs: dict) -> str:
        """Raw accumulator dump of every computed site, line-compatible with the oracle's dump
        (``S``/``A``/``L``/``K``/``Q``/``D`` records).  ``pushed``: the admitted reads in push order;
        ``refs``: tid -> (win_beg, bytes)."""
        out: List[str] = []
        per_lib = self.n_rows > 1 or getattr(self, "_per_lib", False)
        for g in self.regions:
            queues = [[] for _ in range(self.n_rows)]   # site-list semantics: fresh queue per region
            self._dump_region(g, pushed, refs, out, queues, per_lib)
        return "".join(out)

    def dump_range(self, pushed: ReadBatch, refs: dict, region_index: int, pos_lo: int, pos_hi: int, read_offset: int = 0) -> str:
        """Dump of the sites [pos_lo, pos_hi) of one region, starting with an empty deletion queue — what the oracle prints for
        the region (pos_lo+1, pos_hi) whose halo is pos_lo.  ``pushed`` may be a suffix of the pushed stream: ``read_offset`` is the
        stream index of its first read (insertion alleles are looked up in it)."""
        g = dict(self.regions[region_index])
        s0 = pos_lo - g["first_pos"]
        assert 0 <= s0 and pos_hi <= g["first_pos"] + g["n_slots"]
        g["slot_base"] += s0
        g["first_pos"] = pos_lo
        g["n_slots"] = pos_hi - pos_lo
        out: List[str] = []
        self._read_offset = read_offset
        try:
            self._dump_region(g, pushed, refs, out, [[] for _ in range(self.n_rows)], self.n_rows > 1 or getattr(self, "_per_lib", False))
        finally:
            self._read_offset = 0
        return "".join(out)

    def _stat_str(self, v) -> str:
        return " ".join((f"{int(x):08x}" if k in _FLOAT_STATS else str(int(x))) for k, x in enumerate(v))

    def _keys(self, row, slot, pos, pushed, refs, tid):
        bases, indels = {}, []
        if self.pbase[row, slot] < 6:
            bases[int(self.pbase[row, slot])] = self.pstats[:, row, slot]
        j = int(self.sec_head[row, slot])
        while j >= 0:
            k = int(self.sec_kind[j])
            st = self.sec_stats[:, j]
            if k < 6:
                bases[k] = st
            else:
                ln = int(self.sec_len[j])
                if k == KIND_INS:
                    rd, qp = int(self.sec_read[j]) - getattr(self, "_read_offset", 0), int(self.sec_qpos[j])
                    so = int(pushed.seq_off[rd])
                    al = "+"
                    for t in range(1, ln + 1):
                        i = qp + t
                        b = int(pushed.seq[so + (i >> 1)])
                        al += NT[_CANON[(b & 15) if (i & 1) else (b >> 4)]]
                else:
                    wb, seq = refs[tid]
                    al = "-" + seq[pos + 1 - wb: pos + 1 - wb + ln].decode("latin-1")
                indels.append((al.encode("latin-1"), al, st))
            j = int(self.sec_next[j])
        indels.sort(key=lambda x: x[0])
        return bases, indels

    def _dump_region(self, g, pushed, refs, out, queues, per_lib):
        tid = g["tid"]
        for s in range(g["n_slots"]):
            slot = g["slot_base"] + s
            pos = g["first_pos"] + s
            nc = self.ncover[:, slot]
            if (self.flags[:, slot] & 1).any():
                out.append(f"A {tid} {pos}\n")
                continue
            if int(nc.sum()) == 0:
                continue
            mapq_n = int(self.npass[:, slot].sum())
            out.append(f"S {tid} {pos} {int(nc.sum())} {mapq_n}\n")
            extra = 0
            for row in range(self.n_rows):
                if nc[row] == 0:
                    continue
                out.append(f"L {row} {int(nc[row])}\n")
                bases, indels = self._keys(row, slot, pos, pushed, refs, tid)
                for b in range(6):
                    if b in bases and int(bases[b][0]) > 0:
                        out.append(f"K {row} {NT[b]} {self._stat_str(bases[b])}\n")
                for _, al, st in indels:
                    out.append(f"K {row} {al} {self._stat_str(st)}\n")
                    if al[0] == "-":
                        queues[row].append((pos + 1, al, st))
                q = queues[row]
                while q and q[0][0] < pos:
                    q.pop(0)
                while q and q[0][0] == pos:
                    _, al, st = q.pop(0)
                    out.append(f"Q {row} {al} {self._stat_str(st)}\n")
                    extra += int(st[0])
            out.append(f"D {mapq_n + extra}\n")


class PackedResults:
    """Host copy of the PACKED records (include/brc_engine.h): 8 words per (row, slot) + 72-byte secondary records."""

    def __init__(self, r: CPackedResults):
        self.n_rows, self.n_slots = int(r.n_rows), int(r.n_slots)
        rs = self.n_rows * self.n_slots
        self.words = _np_view(r.words, rs * N_WORDS, np.uint32).reshape(N_WORDS, self.n_rows, self.n_slots).copy()
        self.n_sec = int(r.n_sec)
        self.sec = _np_view(r.sec, self.n_sec * (SEC_RECORD_BYTES // 4), np.uint32).reshape(self.n_sec, SEC_RECORD_BYTES // 4).copy()

    def nbytes(self) -> int:
        return int(self.words.nbytes + self.sec.nbytes)

    def widen(self):
        """numpy restatement of the engine's ensure_wide(): (ncover, npass, flags, pbase, pstats[13]) per (row, slot);
        escaped sites are filled from their pool record."""
        w = self.words
        ncover = (w[0] & 0xFF).astype(np.uint32)
        npass = ((w[0] >> 8) & 0xFF).astype(np.uint32)
        count = ((w[0] >> 16) & 0xFF).astype(np.uint32)
        plus = (w[0] >> 24).astype(np.uint32)
        pc = (w[1] & 7).astype(np.uint8)
        flags = ((w[1] >> 3) & 1).astype(np.uint8)
        pbase = np.where(pc < 6, pc, NO_BASE).astype(np.uint8)
        ps = np.stack([count, w[1] >> 16, w[2] & 0xFFFF, w[2] >> 16, plus, count - plus, w[4], w[5], w[3] >> 16, (w[1] >> 8) & 0xFF,
                       w[6], w[3] & 0xFFFF, w[7]]).astype(np.uint32)
        for j in range(self.n_sec):
            rec = self.sec[j]
            kind = int(rec[2]) & 0xFF
            if kind < 8:
                continue
            row, slot = divmod(int(rec[0]), self.n_slots)
            ncover[row, slot] = int(rec[2]) >> 8
            npass[row, slot] = rec[4]
            flags[row, slot] = int(rec[3]) & 1
            pbase[row, slot] = kind - 8 if kind - 8 < 6 else NO_BASE
            ps[:, row, slot] = rec[5:18]
        return ncover, npass, flags, pbase, ps


class SelectedResults:
    """Host copy of a filtered run's sparse results (brc_get_selected_results): the shipped sites' global slot ids (ascending),
    their emit bytes (1 = the line passes, 2 = shipped for the deletion queue, 0 = context), packed words
    [N_WORDS][rows][n_sites] and secondary records (slot = row * n_sites + index into ``site``)."""

    def __init__(self, r: CSelectedResults):
        self.n_rows, self.n_slots, self.n_sites = int(r.n_rows), int(r.n_slots), int(r.n_sites)
        self.regions = [dict(tid=g.tid, beg=g.beg, end=g.end, site_list_mode=g.site_list_mode, slot_base=g.slot_base,
                             first_pos=g.first_pos, n_slots=g.n_slots) for g in (r.regions[i] for i in range(int(r.n_regions)))]
        n = self.n_sites
        self.site = _np_view(r.site, n, np.uint32).copy()
        self.emit = _np_view(r.emit, n, np.uint8).copy()
        self.words = _np_view(r.words, self.n_rows * n * N_WORDS, np.uint32).reshape(N_WORDS, self.n_rows, n).copy()
        self.n_sec = int(r.n_sec)
        self.sec = _np_view(r.sec, self.n_sec * (SEC_RECORD_BYTES // 4), np.uint32).reshape(self.n_sec, SEC_RECORD_BYTES // 4).copy()

    def nbytes(self) -> int:
        """What crossed PCIe for these results: site ids, emit bytes, words and records."""
        return int(self.site.nbytes + self.emit.nbytes + self.words.nbytes + self.sec.nbytes)

    def positions(self, emit: int = 1):
        """0-based reference positions of the sites with the given emit byte, in slot order."""
        starts = np.array([g["slot_base"] for g in self.regions], dtype=np.int64)
        s = self.site[self.emit == emit].astype(np.int64)
        g = np.searchsorted(starts, s, side="right") - 1                 # last region starting at or before the slot
        first = np.array([g_["first_pos"] for g_ in self.regions], dtype=np.int64)
        return (first[g] + s - starts[g]).tolist()


class Engine:
    """One engine handle == one bam-readcount "process" on one GPU."""

    def __init__(self, *, min_mapq=0, min_bq=0, max_cnt=10_000_000, per_lib=False, insertion_centric=False,
                 lib_names: Sequence[str] = (), device: int = 0):
        self.lib = load_library()
        self.lib_names = list(lib_names)
        self.per_lib = bool(per_lib)
        cfg = Config(min_mapq, min_bq, max_cnt, int(per_lib), int(insertion_centric), len(self.lib_names), device, 0)
        h = C.c_void_p()
        rc = self.lib.brc_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise BrcError(rc, self.lib.brc_strerror(rc).decode())
        self.h = h
        self._refs = {}
        self._pushed: List[ReadBatch] = []
        self._keep: list = []
        self._names_arr = (C.c_char_p * max(1, len(self.lib_names)))(*[s.encode() for s in self.lib_names])

    def close(self):
        if getattr(self, "h", None):
            self.lib.brc_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise BrcError(rc, self.lib.brc_last_error(self.h).decode() or self.lib.brc_strerror(rc).decode())

    def set_reference(self, tid: int, name: str, chrom_len: int, seq: bytes, win_beg: int = 0):
        self._check(self.lib.brc_set_reference(self.h, tid, name.encode(), chrom_len, win_beg, seq, len(seq)))
        self._refs[tid] = (win_beg, seq)

    def reset(self):
        self._check(self.lib.brc_reset(self.h))
        self._pushed = []
        self._keep = []

    def begin_region(self, tid: int, beg: int, end: int, site_list_mode: bool = True):
        self._check(self.lib.brc_begin_region(self.h, tid, beg, end, int(site_list_mode)))

    @staticmethod
    def c_batch(b: ReadBatch, keep: list) -> CReadBatch:
        arrs = [np.ascontiguousarray(a) for a in (b.tid, b.pos, b.flag, b.mapq, b.lib, b.l_qseq, b.nm, b.sm, b.cigar_off,
                                                   b.cigar, b.seq_off, b.seq, b.qual_off, b.qual)]
        keep.extend(arrs)
        return CReadBatch(b.n_reads, *[a.ctypes.data for a in arrs])

    def push_reads(self, b: ReadBatch):
        """Bulk push.  The engine may BORROW the arrays (zero-copy) until compute()/reset(), so they are kept
        alive here; pass pinned arrays (``pin_batch``) for full-speed DMA."""
        keep: list = []
        cb = self.c_batch(b, keep)
        self._keep.append(keep)
        self._check(self.lib.brc_push_reads(self.h, C.byref(cb)))

    # ---- f-2: compressed BGZF span -> device-decoded reads -------------------------------------------------
    def _c_span(self, span: dict):
        comp = np.frombuffer(span["comp"], dtype=np.uint8)
        ent = np.asarray(span["entries"], dtype=np.uint64)
        rg = list(span.get("rg_lib", {}).items())
        ids = (C.c_char_p * max(1, len(rg)))(*[k.encode() for k, _ in rg])
        libs = np.asarray([v for _, v in rg] or [0], dtype=np.uint16)
        cs = CBamSpan(comp.ctypes.data, comp.size, ent.size, ent.ctypes.data, int(span.get("end_voff", -1)), int(span["tid"]), len(rg),
                      C.cast(ids, C.c_void_p), libs.ctypes.data)
        return cs, (comp, ent, ids, libs)

    def push_bam_span(self, span: dict):
        """The open region's reads as a compressed BGZF span (bamio.bam_span): inflated and framed on the device."""
        cs, keep = self._c_span(span)
        self._keep.append(keep)
        self._check(self.lib.brc_push_bam_span(self.h, C.byref(cs)))

    def decode_bam_span(self, span: dict) -> ReadBatch:
        """Decode only, and copy the batch back to the host (tests: device decoder == host decoder)."""
        cs, keep = self._c_span(span)
        dev = CReadBatch()
        self._check(self.lib.brc_decode_bam_span(self.h, C.byref(cs), C.byref(dev), None))
        hb = CReadBatch()
        self._check(self.lib.brc_fetch_decoded_batch(self.h, C.byref(hb)))
        n = int(hb.n_reads)
        co = _np_view(hb.cigar_off, n + 1, np.uint64).copy()
        so = _np_view(hb.seq_off, n + 1, np.uint64).copy()
        qo = _np_view(hb.qual_off, n + 1, np.uint64).copy()
        return ReadBatch(tid=np.full(n, int(span["tid"]), np.int32), pos=_np_view(hb.pos, n, np.int32).copy(), flag=_np_view(hb.flag, n, np.uint16).copy(),
                         mapq=_np_view(hb.mapq, n, np.uint8).copy(), lib=_np_view(hb.lib, n, np.uint16).copy(), l_qseq=_np_view(hb.l_qseq, n, np.int32).copy(),
                         nm=_np_view(hb.nm, n, np.int32).copy(), sm=_np_view(hb.sm, n, np.int32).copy(), cigar_off=co,
                         cigar=_np_view(hb.cigar, int(co[n]) if n else 0, np.uint32).copy(), seq_off=so, seq=_np_view(hb.seq, int(so[n]) if n else 0, np.uint8).copy(),
                         qual_off=qo, qual=_np_view(hb.qual, int(qo[n]) if n else 0, np.uint8).copy(), qname=None)

    def end_region(self):
        self._check(self.lib.brc_end_region(self.h))

    def compute(self) -> Optional[Results]:
        self._check(self.lib.brc_compute(self.h))
        if getattr(self, "filtered", False):
            return None
        r = CResults()
        self._check(self.lib.brc_get_results(self.h, C.byref(r)))
        res = Results(r)
        res._per_lib = self.per_lib
        return res

    def warnings(self):
        out = (C.c_int64 * 4)()
        self._check(self.lib.brc_get_warning_counts(self.h, out))
        return tuple(int(x) for x in out)

    def format_text(self, region: int = -1) -> str:
        n = self.lib.brc_format_text(self.h, region, self._names_arr, None, 0)
        if n < 0:
            self._check(int(n))
        buf = C.create_string_buffer(int(n) + 1)
        self.lib.brc_format_text(self.h, region, self._names_arr, buf, int(n) + 1)
        return buf.raw[:int(n)].decode("latin-1")

    # ---- device-resident path (include/brc_engine.h "device-resident path") ---------------------------------
    def set_reference_device(self, tid: int, name: str, chrom_len: int, win_beg: int, dev_ascii_ptr: int, win_len: int, stream_ptr: int):
        self._check(self.lib.brc_set_reference_device(self.h, tid, name.encode(), chrom_len, win_beg, dev_ascii_ptr, win_len, stream_ptr))

    def plan_device(self, regions: Sequence[CRegion], n_reads_cap: int, n_sec_cap: int = 0):
        arr = (CRegion * len(regions))(*regions)
        self._plan_keep = arr
        self._check(self.lib.brc_plan_device(self.h, arr, len(regions), n_reads_cap, n_sec_cap))

    def run_device(self, cbatch: CReadBatch, region_of_read_ptr: Optional[int], stream_ptr: int):
        self._check(self.lib.brc_run_device(self.h, C.byref(cbatch), region_of_read_ptr, stream_ptr))

    def device_packed(self) -> CPackedResults:
        r = CPackedResults()
        self._check(self.lib.brc_device_packed_results(self.h, C.byref(r)))
        return r

    def fetch_device_results(self, stream_ptr: int) -> Optional[Results]:
        self._check(self.lib.brc_fetch_device_results(self.h, stream_ptr))
        if getattr(self, "filtered", False):
            return None
        r = CResults()
        self._check(self.lib.brc_get_results(self.h, C.byref(r)))
        res = Results(r)
        res._per_lib = self.per_lib
        return res

    def packed(self) -> "PackedResults":
        r = CPackedResults()
        self._check(self.lib.brc_get_packed_results(self.h, C.byref(r)))
        return PackedResults(r)

    # ---- alternative-allele site filter (include/brc_engine.h brc_set_site_filter) ----------------------------------------
    def set_site_filter(self, min_alt_count: int, min_alt_fraction: float = 0.0):
        """Print only lines with an alternative allele of count >= min_alt_count and >= min_alt_fraction * depth (from the next
        compute() on); while set, compute() returns None (no dense view) and selected() is the sparse result."""
        f = CSiteFilter(int(min_alt_count), 0, float(min_alt_fraction))
        self._check(self.lib.brc_set_site_filter(self.h, C.byref(f)))
        self.filtered = True

    def clear_site_filter(self):
        self._check(self.lib.brc_set_site_filter(self.h, None))
        self.filtered = False

    def selected(self) -> SelectedResults:
        r = CSelectedResults()
        self._check(self.lib.brc_get_selected_results(self.h, C.byref(r)))
        return SelectedResults(r)

    def stage_ms(self, stage: int) -> float:
        return float(self.lib.brc_last_stage_ms(self.h, stage))

    def launch_count(self) -> int:
        return int(self.lib.brc_last_launch_count(self.h))

    def h2d_bytes(self) -> int:
        """Bytes the last compute() of pushed host reads copied host->device."""
        return int(self.lib.brc_last_h2d_bytes(self.h))


def admitted(batch: ReadBatch, tid: int, max_cnt: int) -> np.ndarray:
    """Indices of the reads of ``batch`` (one region's fetch, file order) the engine keeps — the
    host-side admission rule of brc_push_read (bam_plp_push).  Only used to index results
    (sec_read) back into the caller's batch; the engine applies the same rule itself."""
    import heapq
    end = batch.ref_end()
    it_tid, it_pos = 0, 0
    live: list = []
    keep = []
    for i in range(batch.n_reads):
        t, p, f = int(batch.tid[i]), int(batch.pos[i]), int(batch.flag[i])
        if t < 0 or (f & 4):
            continue
        e = int(end[i])
        if it_tid == t and it_pos == p:
            while live and live[0] < it_pos:
                heapq.heappop(live)
            if len(live) + 1 > max_cnt:
                continue
        linked = e > it_pos or t > it_tid
        if t > it_tid:
            live = []
        it_tid, it_pos = t, p
        if not linked:
            continue
        heapq.heappush(live, e)
        if t == tid:
            keep.append(i)
    return np.array(keep, dtype=np.int64)


def pin_batch(b: ReadBatch) -> ReadBatch:
    """Copy a batch into page-locked host memory (torch's pinned allocator) so brc_compute's H2D copies
    run at full PCIe speed straight out of the caller's buffers."""
    import torch

    def pin(a):
        a = np.ascontiguousarray(a)
        view = {np.dtype(np.uint16): np.int16, np.dtype(np.uint32): np.int32, np.dtype(np.uint64): np.int64}.get(a.dtype)
        t = torch.from_numpy(a.view(view) if view else a).pin_memory()
        out = t.numpy()
        out = out.view(a.dtype) if view else out
        _PINNED_KEEPALIVE.append(t)
        return out
    return ReadBatch(tid=pin(b.tid), pos=pin(b.pos), flag=pin(b.flag), mapq=pin(b.mapq), lib=pin(b.lib), l_qseq=pin(b.l_qseq),
                     nm=pin(b.nm), sm=pin(b.sm), cigar_off=pin(b.cigar_off), cigar=pin(b.cigar), seq_off=pin(b.seq_off),
                     seq=pin(b.seq), qual_off=pin(b.qual_off), qual=pin(b.qual), qname=b.qname)


_PINNED_KEEPALIVE: list = []
