"""The device read generator (csrc/brc_synth.cu, synth_fill_kernel) against the host generator, field for field.

GPU: windows of every shape the fill handles — a full C4 window, the clamped last window of a contig, windows from block 0 and
from lo > 0, DEEP windows whose last CTA is partial with 1, 3 and 8 libraries, with and without region_of_read — are generated on
the device and compared byte for byte with ``Spec.window_host``.  CPU: the same windows (all but the C4 one) exercise every branch
of a read's body — each CIGAR kind, Q2 tails of length 1 and 19, six substitutions, a repeated substitution position and a
substitution drawn on an inserted or clipped base — counted by a numpy restatement of the header draw whose NM, CIGAR kind and
tails are checked against the host generator's output.
"""
import numpy as np
import pytest

from bam_readcount_b200 import synth_cb as sc

FIELDS = ("pos", "flag", "mapq", "lib", "l_qseq", "nm", "sm", "cigar_off", "cigar", "seq_off", "seq", "qual_off", "qual")

C4 = (sc.Spec(seed=1234, contig_len=97656 * sc.BLOCK_BP, n_contigs=24), 0, 0, -(-97656 // 10))
# (spec, contig, lo, hi, with_region)
WINDOWS = [
    (sc.Spec(seed=77, contig_len=1280 * 800, n_contigs=3), 1, 0, 300, True),          # from block 0
    (sc.Spec(seed=78, contig_len=1280 * 800, n_contigs=3), 2, 500, 800, True),        # lo > 0, the contig's last window (starts clamp)
    (sc.Spec(seed=9, contig_len=1280 * 64, n_contigs=1), 0, 60, 64, False),
    (sc.Spec(seed=5, mode=sc.DEEP, n_libs=1, depth=1000, site_stride=700, n_sites=40, contig_len=1280), 3, 27, 40, True),
    (sc.Spec(seed=6, mode=sc.DEEP, n_libs=3, depth=777, site_stride=300, n_sites=40, contig_len=1280), 0, 1, 40, False),
    (sc.Spec(seed=7, mode=sc.DEEP, n_libs=8, depth=50_000, site_stride=1000, n_sites=10, contig_len=1280), 0, 2, 4, True),
    (sc.Spec(seed=8, mode=sc.DEEP, n_libs=8, depth=3, site_stride=5000, n_sites=100, contig_len=1280), 0, 0, 100, True),
]

_M = (1 << 64) - 1


def _u(x):
    return np.uint64(x & _M)


def _mix64(x):
    x = x ^ (x >> _u(30)); x = x * _u(0xbf58476d1ce4e5b9)
    x = x ^ (x >> _u(27)); x = x * _u(0x94d049bb133111eb)
    return x ^ (x >> _u(31))


def _ref_off(kind, q):
    return np.select([kind == 0, kind == 1, kind == 2], [q, np.where(q < 70, q, np.where(q < 72, -1, q - 2)), np.where(q < 60, q, q + 3)],
                     np.where(q < 10, -1, q - 10))


def read_identities(spec, lo, hi, unit):
    """(blk, j) of every read of the window in file order, the WGS blocks sorted by (start, j) as the generator does."""
    if spec.mode == sc.DEEP:
        idx = np.arange(spec.window_reads(lo, hi), dtype=np.int64)
        return (lo + idx // spec.depth).astype(np.uint64), (idx % spec.depth).astype(np.uint64)
    blk = np.repeat(np.arange(lo, hi, dtype=np.int64), sc.BLOCK_READS)
    j = np.tile(np.arange(sc.BLOCK_READS, dtype=np.int64), hi - lo)
    h0 = _stream(_read_key(spec.c.seed, unit, blk.astype(np.uint64), j.astype(np.uint64)), 0)
    start = np.minimum(blk * sc.BLOCK_BP + (h0 & _u(0xFFFFFFFF)).astype(np.int64) % sc.BLOCK_BP, max(spec.contig_len - sc.MAX_SPAN, 0))
    order = np.lexsort((j, start - blk * sc.BLOCK_BP, blk))
    return blk[order].astype(np.uint64), j[order].astype(np.uint64)


def _read_key(seed, unit, blk, j):
    with np.errstate(over="ignore"):
        a = _mix64(np.array([(seed + 0x9E3779B97F4A7C15 * (unit + 1)) & _M], dtype=np.uint64))
        return _mix64(a ^ (blk * _u(0xD1B54A32D192ED03) + j * _u(0x8CB92BA72F3D8DD7) + _u(0x632BE59BD9B4E019)))


def _stream(rk, s):
    with np.errstate(over="ignore"):
        return _mix64(rk + _u((s + 1) * 0xA24BAED4963EE407))


def body_branches(spec, contig, lo, hi):
    """Counts of the read-body branches the window takes, from a restatement of the header and substitution draws; the host
    generator's CIGAR kinds, Q2 tails and NM are asserted to be what the restatement predicts."""
    unit = 0 if spec.mode == sc.DEEP else contig
    batch, _ = spec.window_host(contig, lo, hi)
    n = batch.n_reads
    blk, j = read_identities(spec, lo, hi, unit)
    rk = _read_key(spec.c.seed, unit, blk, j)
    h0, h1, h2, h3 = (_stream(rk, s) for s in range(4))
    kk = ((h0 >> _u(32)) & _u(0xFFFF)).astype(np.int64)
    kind = np.select([kk < 58982, kk < 60948, kk < 62914], [0, 1, 2], 3)
    reverse = ((h0 >> _u(48)) & _u(1)).astype(bool)
    tail = np.where(~reverse & ((h1 & _u(0xFFFF)).astype(np.int64) < 13107), 1 + ((h1 >> _u(16)) & _u(0xFFFF)).astype(np.int64) % 19, 0)
    u = ((h1 >> _u(32)) & _u(0xFFFF)).astype(np.int64)
    n_subs = np.searchsorted(np.array([30898, 54188, 62908, 65069, 65469, 65527]), u, side="right")
    seen = np.full((n, 6), -1, np.int64)
    applied = np.zeros(n, np.int64)
    dup_any = np.zeros(n, bool)
    clip_any = np.zeros(n, bool)
    for t in range(6):
        src = (h2 >> _u(20 * t)) if t < 3 else (h3 >> _u(20 * (t - 3)))
        p = (src & _u(0xFFFF)).astype(np.int64) % 150
        active = t < n_subs
        dup = (seen == p[:, None]).any(axis=1) & active
        new = active & ~dup
        seen[new, t] = p[new]
        clipped = new & (_ref_off(kind, p) < 0)
        applied += new & ~clipped
        dup_any |= dup
        clip_any |= clipped
    # the restatement is the host generator's draw
    n_cig = np.diff(batch.cigar_off.astype(np.int64))
    assert np.array_equal(n_cig, np.select([kind == 0, kind == 3], [1, 2], 3))
    assert np.array_equal(batch.nm, applied + np.select([kind == 1, kind == 2], [2, 3], 0))
    assert np.array_equal(batch.flag, np.where(reverse, 16, 0))
    ql = batch.qual.reshape(n, 150)
    has_tail = tail > 0
    assert (ql[has_tail][np.arange(150)[None, :] >= 150 - tail[has_tail][:, None]] == 2).all()
    return {"kind": np.bincount(kind, minlength=4), "tail1": int((tail == 1).sum()), "tail19": int((tail == 19).sum()),
            "subs6": int((n_subs == 6).sum()), "dup_pos": int(dup_any.sum()), "sub_on_clipped": int(clip_any.sum()),
            "partial_last_cta": n % sc.BLOCK_READS != 0}


def test_windows_cover_every_body_branch():
    tot = {"kind": np.zeros(4, np.int64), "tail1": 0, "tail19": 0, "subs6": 0, "dup_pos": 0, "sub_on_clipped": 0}
    partial_libs = set()
    for sp, contig, lo, hi, _ in WINDOWS:
        c = body_branches(sp, contig, lo, hi)
        for k in tot:
            tot[k] = tot[k] + c[k]
        if c["partial_last_cta"]:
            partial_libs.add(sp.n_libs)
    assert (tot["kind"] > 0).all(), tot
    for k in ("tail1", "tail19", "subs6", "dup_pos", "sub_on_clipped"):
        assert tot[k] > 0, (k, tot)
    assert {1, 3, 8} <= partial_libs
    # the last window of a contig has clamped starts
    sp, contig, lo, hi, _ = WINDOWS[1]
    b, _ = sp.window_host(contig, hi - 1, hi)
    assert (b.pos == sp.contig_len - sc.MAX_SPAN).any()


def _device_equals_host(sp, contig, lo, hi, with_region, dev):
    import torch
    n = sp.window_reads(lo, hi)
    dw = sc.DeviceWindow(sp, n + 300, dev, with_region=with_region)
    for k in ("seq", "qual", "cigar", "region"):          # stale bytes must not survive a fill
        dw.t[k].fill_(0xA5 if dw.t[k].dtype == torch.uint8 else -7)
    dw.fill(contig, lo, hi, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    d = dw.to_host()
    h, ror = sp.window_host(contig, lo, hi)
    for f in FIELDS:
        assert np.array_equal(getattr(d, f), getattr(h, f)), (f, lo, hi)
    if with_region:
        assert np.array_equal(dw.t["region"][:n].cpu().numpy(), ror)


@pytest.mark.gpu
@pytest.mark.parametrize("w", range(len(WINDOWS)))
def test_device_window_equals_host_window(w):
    import torch
    _device_equals_host(*WINDOWS[w], torch.device("cuda", 0))


@pytest.mark.gpu
def test_device_c4_window_equals_host_window():
    import torch
    sp, contig, lo, hi = C4
    _device_equals_host(sp, contig, lo, hi, True, torch.device("cuda", 0))
