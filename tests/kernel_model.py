"""What the kernels decide, restated on the host: their capacities parsed out of csrc/, K0's staged blocks, the tiles' read
ranges and the producer's chunk cuts.  The boundary, pipeline and 32-bit-edge tests use it to assert that a case reaches the
path it claims to."""
from __future__ import annotations

import functools
import os
import re

import numpy as np

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "bam_readcount_b200", "csrc")

CONST_NAMES = ("TILE", "STAGE_READS", "STAGE_QUAL", "STAGE_SEQ", "STAGE_CIGAR", "K0_READS", "K0_QUAL_CAP", "K0_SEQ_CAP", "K0_REF_CAP",
               "FASTDIV_MAX", "DEEP_THREADS", "DEEP_ICACHE", "SEL_LAST_ROWS", "SCAN_CTA")


@functools.lru_cache(maxsize=None)
def kernel_constants():
    """constexpr int NAME = <expression over earlier names>; from csrc/ (BRC_STAGE_READS from its #define)."""
    src = "".join(open(os.path.join(CSRC, f)).read() for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh", ".h")))
    env = {}
    m = re.search(r"#define\s+BRC_STAGE_READS\s+(\d+)", src)
    env["BRC_STAGE_READS"] = int(m.group(1))
    for name in CONST_NAMES:
        m = re.search(r"constexpr\s+int\s+" + name + r"\s*=\s*([^;]+);", src)
        assert m, f"{name} not found in csrc/"
        env[name] = int(eval(m.group(1), {}, dict(env)))
    return env


def k0_m_ops(batch, i, contig, site_list):
    """K0's walk of read i's M ops (read_precompute_kernel): per M op it reaches, (read_position, wrel, j, jend, hit_nul).
    Bases [j, jend) of the op are compared with the reference; those outside the supplied window count as 'N'.  The walk stops
    after an op that reaches the reference's NUL at chrom_len (hit_nul); in site-list mode an op starting past chrom_len
    compares nothing and the walk goes on (R:bamreadcount.cpp:144-151)."""
    _, chrom_len, seq, wb = contig
    co = batch.cigar_off
    ref_pos, rp, out = int(batch.pos[i]), 0, []
    for c in batch.cigar[int(co[i]):int(co[i + 1])].tolist():
        l, op = c >> 4, c & 15
        if op == 0:
            jn, hit = l, False
            if ref_pos + l > chrom_len:
                if site_list and ref_pos > chrom_len:
                    jn = 0
                else:
                    jn, hit = max(0, chrom_len - ref_pos), True
            wrel = ref_pos - wb
            j = min(jn, -wrel) if wrel < 0 else 0
            out.append((rp, wrel, j, max(j, min(jn, len(seq) - wrel)), hit))
            if hit:
                break
            ref_pos += l; rp += l
        elif op in (2, 3):
            ref_pos += l
        elif op in (1, 4):
            rp += l
    return out


def k0_launch_blocks(n, launches=None):
    """(r0, r1) of every K0 block: each launch [a, b) covers its reads in blocks of K0_READS from a."""
    K = kernel_constants()["K0_READS"]
    return [(r0, min(b, r0 + K)) for a, b in (launches or [(0, n)]) for r0 in range(a, b, K)]


def k0_blocks(batch, case, launches=None, site_list=None, ops=False):
    """Per K0 block of a single-region batch: staged, uniform length, ref staged, an op past the staged reference window, the
    span of its first positions, and with ops=True per read the M ops K0 walks (k0_m_ops) each with `ref_staged`, the
    condition under which K0 reads that op's reference codes from the staged window (brc_kernels.cu, `ref_staged = ...`)."""
    K = kernel_constants()
    contig = case["contigs"][0]
    sl = case["site_list"] if site_list is None else site_list
    win_len, wb = len(contig[2]), contig[3]
    end = batch.ref_end()
    out = []
    for r0, r1 in k0_launch_blocks(batch.n_reads, launches):
        qa, qb = int(batch.qual_off[r0]) & ~15, (int(batch.qual_off[r1]) + 15) & ~15
        sa, sb = int(batch.seq_off[r0]) & ~15, (int(batch.seq_off[r1]) + 15) & ~15
        staged = qb - qa <= K["K0_QUAL_CAP"] and sb - sa <= K["K0_SEQ_CAP"]
        ra = rb = 0
        if staged:
            pf, pl = int(batch.pos[r0]) - wb, int(batch.pos[r1 - 1]) - wb
            nbytes = (win_len + 1) // 2 + 16
            ra = ((pf >> 1) if pf > 0 else 0) & ~15
            rb = min((((pl + 1024) >> 1) + 31) & ~15, nbytes & ~15)
            if rb <= ra or rb - ra > K["K0_REF_CAP"]:
                ra = rb = 0
        past = bool(rb > ra and any(((int(end[i]) - wb) >> 1) + 8 >= rb for i in range(r0, r1)))
        blk = dict(r0=r0, r1=r1, staged=staged, uniform=len(set(batch.l_qseq[r0:r1].tolist())) == 1, lq=int(batch.l_qseq[r0]),
                   ref_staged=rb > ra, past=past, span=int(batch.pos[r1 - 1]) - int(batch.pos[r0]))
        if ops:
            blk["ops"] = [[dict(rp=rp, wrel=wrel, j=j, jend=jend, hit_nul=hit,
                                ref_staged=rb > ra and ((wrel + j) >> 1) >= ra and ((wrel + jend) >> 1) + 8 < rb)
                           for rp, wrel, j, jend, hit in k0_m_ops(batch, i, contig, sl)] for i in range(r0, r1)]
        out.append(blk)
    return out


def _tile_spans(pos, end, first_pos, end_excl):
    """(read, tile) pairs of every read overlapping [first_pos, end_excl) (tile index relative to the region's first tile)."""
    T = kernel_constants()["TILE"]
    a = np.maximum(pos.astype(np.int64), first_pos)
    b = np.minimum(end.astype(np.int64), end_excl)
    idx = np.nonzero(b > a)[0]
    t0 = (a[idx] - first_pos) // T
    cnt = (b[idx] - 1 - first_pos) // T - t0 + 1
    rep = np.repeat(np.arange(idx.shape[0]), cnt)
    step = np.arange(rep.shape[0]) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    return idx[rep], t0[rep] + step


TILE_LO_INIT, TILE_HI_INIT = 0x7FFFFFFF, 0      # init_tiles_kernel: what a tile no read overlaps keeps


def tile_ranges(batch, first_pos, end_excl):
    """tile_lo / tile_hi of one region (K0's atomics): first / one-past-last read overlapping each TILE-site tile."""
    T = kernel_constants()["TILE"]
    n_t = (end_excl - first_pos + T - 1) // T
    lo = np.full(n_t, TILE_LO_INIT, np.int64); hi = np.full(n_t, TILE_HI_INIT, np.int64)
    end = np.where((batch.flag & 4) != 0, batch.pos.astype(np.int64), batch.ref_end())
    r, t = _tile_spans(batch.pos, end, first_pos, end_excl)
    np.minimum.at(lo, t, r); np.maximum.at(hi, t, r + 1)
    return [(int(l), int(h)) if l < h else (0, 0) for l, h in zip(lo, hi)]


# ---- ReadDesc (brc_device.cuh), restated -------------------------------------------------------------------------------------
DESC = np.dtype([("pos", "<i4"), ("end", "<i4"), ("fm", "<u4"), ("lib_nc", "<u4"),
                 ("mmq", "<i4"), ("clen", "<i4"), ("lclip", "<i4"), ("tpi", "<i4"),
                 ("q2", "<i4"), ("nmfrac", "<f4"), ("se", "<i4"), ("fl", "<f4"),
                 ("qual32", "<u4"), ("seq32", "<u4"), ("cig", "<u4"), ("n_cigar", "<u4"),
                 ("rcp_l", "<f4"), ("rcp_clen", "<f4"), ("fclen", "<f4"), ("inc", "<u4")])
assert DESC.itemsize == 80
FM_SIMPLE, FM_NM_ABSENT, FM_SM_MISSING, FM_FASTDIV, FM_HOT, FM_DEAD = (1 << k for k in range(24, 30))
FLAG_FILTER = 4 | 256 | 512 | 1024
TAG_ABSENT = -2 ** 31
INT32_MAX = 2 ** 31 - 1


def cigar_shape(batch):
    """Per read: FM_SIMPLE (exactly one reference-consuming op, of type M, = or X, and no I or P) and qoff (the soft clips
    before the first reference-consuming op), vectorised over the CIGAR pool."""
    n = batch.n_reads
    co = batch.cigar_off.astype(np.int64)
    cig = batch.cigar[co[0]:co[n]]
    ops, lens = cig & 15, (cig >> 4).astype(np.int64)
    read = np.repeat(np.arange(n), np.diff(co))
    is_ref = np.isin(ops, (0, 2, 3, 7, 8))
    n_ref = np.bincount(read, is_ref, n)
    bad = np.bincount(read, (is_ref & ~np.isin(ops, (0, 7, 8))) | np.isin(ops, (1, 6)), n)
    excl = np.concatenate([[0], np.cumsum(is_ref)])            # excl[k]: reference-consuming ops before op k of the pool
    ref_before = excl[:-1] - np.repeat(excl[co[:-1] - co[0]], np.diff(co))
    qoff = np.zeros(n, np.int64)
    s = (ops == 4) & (ref_before == 0)
    np.add.at(qoff, read[s], lens[s])
    return (n_ref == 1) & (bad == 0), qoff


def _f32_div(a, b, where):
    out = np.zeros(a.shape[0], np.float32)
    np.divide(a.astype(np.float32), b.astype(np.float32), out=out, where=where)
    return out


def k0_descriptors(batch, regions, refs, flags, offsets=None):
    """The read descriptors and tile ranges K0 writes for ``batch`` (the reads as the engine holds them, in its order).

    regions  per region, in tile order: dict(ref=index into refs, site_list, first_pos, n_slots, read_lo, read_hi)
    refs     (name, chrom_len, window bytes, win_beg) per contig, as given to brc_set_reference
    flags    the engine's flags (min_mapq)
    offsets  {"cigar", "seq", "qual": n+1 offsets} of the pools the engine used (default: the batch's own)
    Returns (desc as a DESC array, tile_lo, tile_hi) in the shapes Engine.read_descriptors() returns them, viewed as DESC.
    fetch_func's five values and bam_endpos come from the oracle (oracle.read_values); the rest restates brc_device.cuh."""
    from oracle.oracle import read_values
    K = kernel_constants()
    n = batch.n_reads
    off = {k: batch_off.astype(np.uint64) for k, batch_off in
           (("cigar", batch.cigar_off), ("seq", batch.seq_off), ("qual", batch.qual_off))}
    off.update({k: np.asarray(v, np.uint64) for k, v in (offsets or {}).items()})
    d = np.zeros(n, DESC)
    end = np.zeros(n, np.int64)
    for g in regions:
        lo, hi = g["read_lo"], g["read_hi"]
        v = read_values(batch, refs[g["ref"]], g["site_list"], lo, hi)
        d["mmq"][lo:hi], d["clen"][lo:hi], d["lclip"][lo:hi], d["tpi"][lo:hi], d["q2"][lo:hi] = v[:5]
        end[lo:hi] = v.endpos
    flag = batch.flag.astype(np.uint32); mapq = batch.mapq.astype(np.uint32)
    lq, clen, nm, sm = batch.l_qseq, d["clen"], batch.nm, batch.sm
    end = np.where(flag & 4, batch.pos.astype(np.int64), end)      # never admitted to the pileup: covers nothing
    d["pos"] = batch.pos
    d["end"] = np.minimum(end, INT32_MAX)
    simple, qoff = cigar_shape(batch)
    n_cig = np.diff(batch.cigar_off.astype(np.int64))
    fast = (lq >= 1) & (lq <= K["FASTDIV_MAX"]) & (clen >= 1) & (clen <= K["FASTDIV_MAX"])
    nm_absent = nm == TAG_ABSENT
    sm_missing = ((flag & 2) != 0) & (sm == TAG_ABSENT)
    fm = flag | mapq << 16
    fm |= np.where(simple, FM_SIMPLE, 0).astype(np.uint32)
    fm |= np.where(nm_absent, FM_NM_ABSENT, 0).astype(np.uint32)
    fm |= np.where(sm_missing, FM_SM_MISSING, 0).astype(np.uint32)
    fm |= np.where(fast, FM_FASTDIV, 0).astype(np.uint32)
    fm |= np.where(simple & fast & ~nm_absent & ~sm_missing, FM_HOT, 0).astype(np.uint32)
    fm |= np.where((mapq.astype(np.int64) < flags.get("min_mapq", 0)) | ((flag & FLAG_FILTER) != 0), FM_DEAD, 0).astype(np.uint32)
    d["fm"] = fm
    d["lib_nc"] = batch.lib.astype(np.uint32) | np.minimum(n_cig, 0xFFFF).astype(np.uint32) << 16
    d["nmfrac"] = _f32_div(nm, clen, ~nm_absent)          # +0 where NM is absent
    d["se"] = np.where(flag & 2, np.where(sm == TAG_ABSENT, 0, sm), mapq.astype(np.int64))
    d["fl"] = lq.astype(np.float32)
    d["qual32"] = off["qual"][:n] & np.uint64(0xFFFFFFFF)
    d["seq32"] = off["seq"][:n] & np.uint64(0xFFFFFFFF)
    d["cig"] = np.where(simple, qoff.astype(np.uint64), off["cigar"][:n] & np.uint64(0xFFFFFFFF))
    d["n_cigar"] = n_cig
    d["rcp_l"] = _f32_div(np.ones(n), lq, fast)
    d["rcp_clen"] = _f32_div(np.ones(n), clen, fast)
    d["fclen"] = clen.astype(np.float32)
    d["inc"] = 1 | np.where(flag & 16, 0, 256) | np.where(d["q2"] > -1, 65536, 0)
    # tile ranges: every region's tiles in tile_base order
    T = K["TILE"]
    n_t = [(g["n_slots"] + T - 1) // T for g in regions]
    tlo = np.full(sum(n_t), TILE_LO_INIT, np.int64); thi = np.full(sum(n_t), TILE_HI_INIT, np.int64)
    base = 0
    for g, nt in zip(regions, n_t):
        lo, hi = g["read_lo"], g["read_hi"]
        r, t = _tile_spans(batch.pos[lo:hi], end[lo:hi], g["first_pos"], g["first_pos"] + g["n_slots"])
        np.minimum.at(tlo, base + t, lo + r); np.maximum.at(thi, base + t, lo + r + 1)
        base += nt
    return d, tlo.astype(np.int32), thi.astype(np.int32)


def k1_chunks(batch, ranges):
    """The producer's chunk cuts (brc_kernels.cu pileup_kernel, warp 8): per chunk (r0, r1, full size, staged, CIGAR ops window,
    CIGAR staged)."""
    K = kernel_constants()
    SQ, SS, SR, SC = K["STAGE_QUAL"], K["STAGE_SEQ"], K["STAGE_READS"], K["STAGE_CIGAR"]
    qo, so, co = (x.astype(np.int64) for x in (batch.qual_off, batch.seq_off, batch.cigar_off))
    out = []
    for lo, hi in ranges:
        r0 = lo
        while r0 < hi:
            r1 = min(r0 + SR, hi)
            full = r1 - r0
            while True:
                qa, qb = int(qo[r0]) & ~15, (int(qo[r1]) + 15) & ~15
                sa, sb = int(so[r0]) & ~15, (int(so[r1]) + 15) & ~15
                staged = qb - qa <= SQ and sb - sa <= SS
                if staged or r1 - r0 == 1:
                    break
                fq, fs = (SQ - 32) / (qb - qa), (SS - 32) / (sb - sa)
                n2 = int((r1 - r0) * min(fq, fs))
                r1 = r0 + max(1, min(n2, r1 - r0 - 1))
            ca, cb = int(co[r0]) & ~3, (int(co[r1]) + 3) & ~3
            out.append(dict(r0=r0, r1=r1, full=full, staged=staged, cops=cb - ca, cstaged=cb - ca <= SC,
                            lq=set(batch.l_qseq[r0:r1].tolist())))
            r0 = r1
    return out
