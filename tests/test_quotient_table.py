"""The quotient tables the pileup kernels read in place of divisions (brc_device.cuh QTAB_*).

  * every entry of every row against numpy's correctly rounded float32 division, and 1 - (double) of it;
  * a C3-sized run (10 Mb, 30x, -q 20 -b 20) gives the same packed records and pool records as a build of the library with
    -DBRC_NO_QTAB, whose kernels divide with the reciprocal and one Newton step instead.
"""
from __future__ import annotations

import os
import subprocess
import sys

import numpy as np
import pytest

from cases import ROOT
pytestmark = pytest.mark.gpu

FASTDIV_MAX, QTAB_MID, QTAB_W = 2048, 2048, 4096


def test_every_table_entry_is_the_correctly_rounded_quotient():
    from bam_readcount_b200.engine import Engine
    e = Engine()
    try:
        q, p = e.quotient_rows(1, FASTDIV_MAX)
    finally:
        e.close()
    d = np.arange(1, FASTDIV_MAX + 1, dtype=np.int64)[:, None]
    j = np.arange(QTAB_W, dtype=np.int64)[None, :] - QTAB_MID
    want_q = np.abs(j).astype(np.float32) / d.astype(np.float32)
    posf = np.abs(2 * j - d).astype(np.float32) / d.astype(np.float32)
    want_p = 1.0 - posf.astype(np.float64)
    bad_q = np.argwhere(q.view(np.uint32) != want_q.view(np.uint32))
    bad_p = np.argwhere(p.view(np.uint64) != want_p.view(np.uint64))
    assert len(bad_q) == 0, f"{len(bad_q)} Q entries differ, first (d, j) = ({bad_q[0][0] + 1}, {bad_q[0][1] - QTAB_MID})"
    assert len(bad_p) == 0, f"{len(bad_p)} P entries differ, first (d, j) = ({bad_p[0][0] + 1}, {bad_p[0][1] - QTAB_MID})"
    # posf, as the kernels recover it from P for the events that are not a site's primary base class
    assert np.array_equal((1.0 - p).astype(np.float32).view(np.uint32), posf.view(np.uint32))


# One C3-sized run through brc_run_device; writes the packed words and the pool records (without the chain link, sorted: pool
# order depends on thread timing) to argv[1].  The library is the one BRC_ENGINE_LIB names, or the in-tree one.
RUN = r"""
import ctypes as C, sys
import numpy as np, torch
from bam_readcount_b200 import synth
from bam_readcount_b200.engine import Engine, CReadBatch, CRegion
L = 10_000_000
ref = synth.synth_reference(L, 1234); batch = synth.synth_reads(ref, 30, seed=1234); n = batch.n_reads
eng = Engine(min_mapq=20, min_bq=20); eng.set_reference(0, "chr1", L, ref.tobytes(), 0)
def dev(a):
    a = np.ascontiguousarray(a)
    v = {np.dtype(np.uint16): np.int16, np.dtype(np.uint32): np.int32, np.dtype(np.uint64): np.int64}.get(a.dtype)
    return torch.from_numpy(a.view(v) if v else a).cuda()
pad = np.zeros(64, np.uint8)
d = dict(pos=dev(batch.pos), flag=dev(batch.flag), mapq=dev(batch.mapq), lib=dev(batch.lib), l_qseq=dev(batch.l_qseq), nm=dev(batch.nm),
         sm=dev(batch.sm), cigar_off=dev(batch.cigar_off), cigar=dev(np.concatenate([batch.cigar, np.zeros(16, np.uint32)])),
         seq_off=dev(batch.seq_off), seq=dev(np.concatenate([batch.seq, pad])), qual_off=dev(batch.qual_off),
         qual=dev(np.concatenate([batch.qual, pad])))
cb = CReadBatch(n, None, *[d[k].data_ptr() for k in ("pos", "flag", "mapq", "lib", "l_qseq", "nm", "sm", "cigar_off", "cigar", "seq_off",
                                                     "seq", "qual_off", "qual")])
eng._check(eng.lib.brc_plan_device(eng.h, C.byref(CRegion(0, 0, L, 0, 0, n, 0, 0, L)), 1, n, 0))
sp = torch.cuda.current_stream().cuda_stream
eng.run_device(cb, None, sp)
eng.fetch_device_results(sp)
pk = eng.packed()
sec = np.delete(pk.sec, 1, axis=1)
sec = sec[np.lexsort(sec.T[::-1])] if len(sec) else sec
np.savez(sys.argv[1], words=pk.words, sec=sec)
"""


def _run(out, env):
    subprocess.run([sys.executable, "-c", RUN, out], cwd=ROOT, env=env, check=True, timeout=900)
    with np.load(out) as z:
        return z["words"], z["sec"]


def test_c3_records_equal_the_division_build(tmp_path):
    from bam_readcount_b200 import build
    lib = str(tmp_path / "libbrc_engine_noqtab.so")
    cmd = [build.nvcc_path()] + build.NVCC_FLAGS + ["-DBRC_NO_QTAB", "-I", os.path.join(ROOT, "include"), "-o", lib] + \
          [os.path.join(build.CSRC, s) for s in build.SOURCES]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout[-4000:]
    env = {k: v for k, v in os.environ.items() if k != "BRC_ENGINE_LIB"}
    w_tab, s_tab = _run(str(tmp_path / "qtab.npz"), env)
    w_div, s_div = _run(str(tmp_path / "div.npz"), dict(env, BRC_ENGINE_LIB=lib))
    assert w_tab.shape == w_div.shape and w_tab.size > 0
    diff = np.argwhere(w_tab != w_div)
    assert len(diff) == 0, f"{len(diff)} packed words differ, first (word, row, slot) = {tuple(diff[0])}"
    assert np.array_equal(s_tab, s_div), "pool records differ"
