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


def k0_blocks(batch, case):
    """(staged, ref staged, an op past the staged reference window) per K0 block of a single-region batch."""
    K = kernel_constants()
    n = batch.n_reads
    name, chrom_len, seq, wb = case["contigs"][0]
    win_len = len(seq)
    end = batch.ref_end()
    out = []
    for r0 in range(0, n, K["K0_READS"]):
        r1 = min(n, r0 + K["K0_READS"])
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
        out.append(dict(staged=staged, uniform=len(set(batch.l_qseq[r0:r1].tolist())) == 1, lq=int(batch.l_qseq[r0]),
                        ref_staged=rb > ra, past=past, span=int(batch.pos[r1 - 1]) - int(batch.pos[r0])))
    return out


def tile_ranges(batch, first_pos, end_excl):
    """tile_lo / tile_hi of one region (K0's atomics): first / one-past-last read overlapping each TILE-site tile."""
    T = kernel_constants()["TILE"]
    n_t = (end_excl - first_pos + T - 1) // T
    lo = np.full(n_t, 2 ** 31 - 1, np.int64); hi = np.zeros(n_t, np.int64)
    e = batch.ref_end()
    for i in range(batch.n_reads):
        if batch.flag[i] & 4:
            continue
        a, b = max(int(batch.pos[i]), first_pos), min(int(e[i]), end_excl)
        if b <= a:
            continue
        for t in range((a - first_pos) // T, (b - 1 - first_pos) // T + 1):
            lo[t] = min(lo[t], i); hi[t] = max(hi[t], i + 1)
    return [(int(l), int(h)) if l < h else (0, 0) for l, h in zip(lo, hi)]


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
