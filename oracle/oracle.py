"""TEST INFRASTRUCTURE — ctypes wrapper around oracle/brc_oracle.c (the CPU restatement).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this.
The product package never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import List, NamedTuple, Optional, Sequence, Tuple

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
BUILD = os.path.join(HERE, "_build")
LIB = os.path.join(BUILD, "liboracle.so")
REF_DIR = os.path.join(HERE, "_ref")
REF_BIN = os.path.join(REF_DIR, "bam-readcount")
REF_SAMTOOLS = os.path.join(REF_DIR, "samtools")
REF_DATA = os.path.join(REF_DIR, "test-data")


def build(force: bool = False) -> str:
    src = os.path.join(HERE, "brc_oracle.c")
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < os.path.getmtime(src):
        os.makedirs(BUILD, exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-std=c99", "-shared", "-fPIC", "-w",
                               "-o", LIB, src, "-lm"])
    return LIB


class _Reads(C.Structure):
    _fields_ = [("n_reads", C.c_int64), ("tid", C.c_void_p), ("pos", C.c_void_p), ("flag", C.c_void_p),
                ("mapq", C.c_void_p), ("lib", C.c_void_p), ("l_qseq", C.c_void_p), ("nm", C.c_void_p),
                ("sm", C.c_void_p), ("cigar_off", C.c_void_p), ("cigar", C.c_void_p), ("seq_off", C.c_void_p),
                ("seq", C.c_void_p), ("qual_off", C.c_void_p), ("qual", C.c_void_p)]


class _Config(C.Structure):
    _fields_ = [("min_mapq", C.c_int32), ("min_bq", C.c_int32), ("max_cnt", C.c_int32), ("per_lib", C.c_int32),
                ("insertion_centric", C.c_int32), ("n_libs", C.c_int32), ("lib_names", C.POINTER(C.c_char_p))]


class _Ref(C.Structure):
    _fields_ = [("tid", C.c_int32), ("name", C.c_char_p), ("chrom_len", C.c_int64), ("win_beg", C.c_int64),
                ("win_len", C.c_int64), ("seq", C.c_char_p)]


_lib = None


def _load():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.orc_ctx_new.restype = C.c_void_p
        _lib.orc_ctx_new.argtypes = [C.c_int]
        _lib.orc_ctx_free.argtypes = [C.c_void_p]
        _lib.orc_ctx_clear_queues.argtypes = [C.c_void_p]
        _lib.orc_ctx_reset_output.argtypes = [C.c_void_p]
        _lib.orc_ctx_text.restype = C.c_void_p
        _lib.orc_ctx_text.argtypes = [C.c_void_p]
        _lib.orc_ctx_dump.restype = C.c_void_p
        _lib.orc_ctx_dump.argtypes = [C.c_void_p]
        _lib.orc_ctx_text_len.restype = C.c_int64
        _lib.orc_ctx_text_len.argtypes = [C.c_void_p]
        _lib.orc_ctx_dump_len.restype = C.c_int64
        _lib.orc_ctx_dump_len.argtypes = [C.c_void_p]
        _lib.orc_ctx_lines.restype = C.c_int64
        _lib.orc_ctx_lines.argtypes = [C.c_void_p]
        _lib.orc_ctx_warnings.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
        _lib.orc_region.restype = C.c_int64
        _lib.orc_region.argtypes = [C.c_void_p, C.POINTER(_Config), C.POINTER(_Ref), C.POINTER(_Reads), C.c_int64,
                                    C.c_int64, C.c_int32, C.c_int64, C.c_int64, C.c_int]
        _lib.orc_read_values.restype = None
        _lib.orc_read_values.argtypes = [C.POINTER(_Ref), C.POINTER(_Reads), C.c_int64, C.c_int64, C.c_int, C.c_void_p,
                                         C.c_void_p]
    return _lib


def _c_reads(b):
    """The batch as orc_reads, and the arrays its pointers point into (keep them alive while it is used)."""
    keep = [np.ascontiguousarray(a) for a in (b.tid, b.pos, b.flag, b.mapq, b.lib, b.l_qseq, b.nm, b.sm, b.cigar_off,
                                               b.cigar, b.seq_off, b.seq, b.qual_off, b.qual)]
    return _Reads(b.n_reads, *[a.ctypes.data for a in keep]), keep


class ReadValues(NamedTuple):
    """fetch_func's per-read values (R:bamreadcount.cpp:114-253) and bam_endpos (V:htslib-1.10/sam.c:507-513)."""
    mmq: np.ndarray            # sum_of_mismatch_qualities, int32
    clipped_length: np.ndarray
    left_clip: np.ndarray
    tpi: np.ndarray            # three_prime_index
    q2_pos: np.ndarray
    endpos: np.ndarray         # int64; pos + 1 for unmapped reads and reads without CIGAR


def read_values(batch, contig, site_list_mode: bool, lo: int = 0, hi: Optional[int] = None) -> ReadValues:
    """fetch_values / read_endpos of reads [lo, hi) of ``batch`` against ``contig`` = (name, chrom_len, window bytes,
    win_beg); ``site_list_mode`` is the reference's ref_len check (-l)."""
    lib = _load()
    hi = batch.n_reads if hi is None else hi
    name, chrom_len, seq, win_beg = contig
    reads, keep = _c_reads(batch)
    ref = _Ref(0, name.encode(), chrom_len, win_beg, len(seq), seq)
    zm = np.zeros((max(hi - lo, 0), 5), np.int32)
    end = np.zeros(max(hi - lo, 0), np.int64)
    if hi > lo:
        lib.orc_read_values(C.byref(ref), C.byref(reads), lo, hi, int(site_list_mode), zm.ctypes.data, end.ctypes.data)
    del keep
    return ReadValues(*(zm[:, k].copy() for k in range(5)), end)


class Oracle:
    """One bam-readcount "process": config + deletion queues that persist across regions."""

    def __init__(self, *, min_mapq=0, min_bq=0, max_cnt=10_000_000, per_lib=False, insertion_centric=False,
                 lib_names: Sequence[str] = ()):
        self.lib = _load()
        self.lib_names = list(lib_names)
        self._names_arr = (C.c_char_p * max(1, len(self.lib_names)))(*[s.encode() for s in self.lib_names])
        self.cfg = _Config(min_mapq, min_bq, max_cnt, int(per_lib), int(insertion_centric), len(self.lib_names),
                           self._names_arr)
        self.n_rows = len(self.lib_names) if per_lib else 1
        self.ctx = self.lib.orc_ctx_new(self.n_rows)

    def __del__(self):
        try:
            if self.ctx:
                self.lib.orc_ctx_free(self.ctx)
                self.ctx = None
        except Exception:
            pass

    def region(self, batch, *, tid: int, beg: int, end: int, contig: str, chrom_len: int, ref_seq: bytes,
               ref_win_beg: int = 0, site_list_mode: bool = True, read_lo: int = 0, read_hi: Optional[int] = None):
        """Run one region: ``beg`` is the reference's d.beg (0-based first printed site), ``end`` its d.end.
        ``batch`` holds (from read_lo to read_hi) the records fetched for [beg-1, end) in file order."""
        b = batch
        reads, keep = _c_reads(b)
        ref = _Ref(tid, contig.encode(), chrom_len, ref_win_beg, len(ref_seq), ref_seq)
        hi = b.n_reads if read_hi is None else read_hi
        n = self.lib.orc_region(self.ctx, C.byref(self.cfg), C.byref(ref), C.byref(reads), read_lo, hi, tid, beg, end,
                                int(site_list_mode))
        if site_list_mode:
            self.lib.orc_ctx_clear_queues(self.ctx)   # R:bamreadcount.cpp:605
        return n

    def text(self) -> str:
        n = self.lib.orc_ctx_text_len(self.ctx)
        return C.string_at(self.lib.orc_ctx_text(self.ctx), n).decode("latin-1")

    def dump(self) -> str:
        n = self.lib.orc_ctx_dump_len(self.ctx)
        return C.string_at(self.lib.orc_ctx_dump(self.ctx), n).decode("latin-1")

    def n_lines(self) -> int:
        return int(self.lib.orc_ctx_lines(self.ctx))

    def warnings(self) -> Tuple[int, int, int]:
        out = (C.c_int64 * 3)()
        self.lib.orc_ctx_warnings(self.ctx, out)
        return tuple(int(x) for x in out)

    def reset_output(self):
        self.lib.orc_ctx_reset_output(self.ctx)


def have_reference_binary() -> bool:
    return os.path.exists(REF_BIN) and os.access(REF_BIN, os.X_OK)


def run_reference_binary(args: List[str], cwd: Optional[str] = None, timeout: Optional[float] = None) -> Tuple[str, str, int]:
    """Run the UNMODIFIED reference binary (oracle/_ref/bam-readcount)."""
    p = subprocess.run([REF_BIN] + args, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=timeout)
    return p.stdout.decode("latin-1"), p.stderr.decode("latin-1"), p.returncode
