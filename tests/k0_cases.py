"""Seeded reads aimed at the edges of K0 (read_precompute_kernel, brc_kernels.cu), for tests/test_k0_descriptors.py.

One contig, one case, its reads in position order, section by section:
  phases    every read-start nibble phase 0-7 in its 32-bit word (set by the soft clip before the first M op) against every
            reference nibble phase 0-7 (set by the position), M ops of 1-49 bases with a mismatch at every lane of a 16-base
            step, runs of adjacent mismatches across a step, across M D M and M N M (adjacent in read coordinates: one run) and
            across M I M (not adjacent)
  codes     all 16 x 16 (read code, reference code) pairs: read '=' (code 0), reference '=', N, IUPAC codes, lower case, the
            digits 0-3 and bytes outside the table (code 15)
  quals     l_qseq 1-12, 150 and 151, every quality offset mod 4 on both strands, Q2 runs of every length up to the whole
            read, every byte value at the byte that stops the scan, soft clips at both ends (each three_prime_index clamp
            binds), H before S, = and X ops, P, H and op 9, a mapped read without CIGAR, flags, tags and libraries
  sparse    a block whose first positions span more than 2 * K0_REF_CAP bases (reference not staged), and a block ending in
            reads whose long D / N carry a later M op past the staged reference window
  long      200-2049 base reads (bases and qualities from global memory), l_qseq and clipped length at FASTDIV_MAX and one
            past it, and a read of more than 65,535 CIGAR ops
  ends      M ops running past the end of the supplied reference window, and past chrom_len: an M op ending inside it,
            one starting exactly at it and one starting past it (the site-list mode skips those positions and walks on)
The quality offset of each read is chosen by padding the previous read's qualities with bytes other than 2, so that the
masks of the Q2 scan have something to mask; the pools of the case are therefore not those a copied push builds.
k0_case(unmapped=True) adds placed unmapped reads among the others, for brc_run_device (a push never admits them).

Out of scope: reads whose SEQ is '*' (l_qseq 0) and that have M ops.  fetch_func then reads bytes outside the record, and no
reference defines what it finds there."""
from __future__ import annotations

import functools

import numpy as np

from bam_readcount_b200.batch import BatchBuilder, parse_cigar_string

# seq_nt16_table (V:htslib-1.10/hts.c:73-91), as the engine encodes the reference
NT16 = np.full(256, 15, np.uint8)
for _i, _c in enumerate("=ACMGRSVTWYHKDBN"):
    NT16[ord(_c)] = NT16[ord(_c.lower())] = _i
for _i, _c in enumerate("0123"):
    NT16[ord(_c)] = 1 << _i
# reference characters of each code 0-15, two spellings each (the second: lower case, a digit, or a byte outside the table)
CODE_CHARS = (b"=ACMGRSVTWYHKDBN", b"=a1m2rsv3wyhkdb*")
WIN_BEG = 1000
CHROM_LEN = 160_000
WIN_END = CHROM_LEN - 300           # the supplied window is [WIN_BEG, WIN_END); printed sites end there too
BASES = np.array([1, 2, 4, 8], np.uint8)
PAD_BYTES = np.array([0x00, 0x01, 0x03, 0x82, 0xFF, 0x22, 40], np.uint8)


class _Builder:
    def __init__(self, seed, unmapped):
        self.rng = np.random.default_rng(seed)
        self.unmapped = unmapped
        ref = self.rng.choice(np.frombuffer(b"ACGT", np.uint8), size=CHROM_LEN)
        messy = self.rng.random(CHROM_LEN) < 0.03
        ref[messy] = self.rng.choice(np.frombuffer(b"NacgtRyn", np.uint8), size=int(messy.sum()))
        self.ref = ref
        self.recs = []

    def codes(self, p, n):
        return NT16[self.ref[p:p + n]] if p + n <= CHROM_LEN else np.concatenate([NT16[self.ref[p:]], np.full(p + n - CHROM_LEN, 15, np.uint8)])

    def add(self, pos, cigar, *, mm=(), read_codes=None, flag=0, mapq=60, lib=0, nm=1, sm=None, qual=None, lead=None, l_qseq=None):
        """One read: its bases copy the reference (a base A/C/G/T where the reference has none) except at the read offsets in
        `mm`, which get another base; `read_codes` gives them outright.  `lead`: its quality offset mod 4."""
        rng = self.rng
        ops = [(int(c) >> 4, int(c) & 15) for c in (parse_cigar_string(cigar) if isinstance(cigar, str) else cigar)]
        if read_codes is None:
            out, rp = [], pos
            for l, o in ops:
                if o in (0, 7, 8):
                    c = self.codes(rp, l).copy()
                    bad = ~np.isin(c, BASES)
                    c[bad] = rng.choice(BASES, size=int(bad.sum()))
                    out.append(c); rp += l
                elif o in (2, 3):
                    rp += l
                elif o in (1, 4):
                    out.append(rng.choice(BASES, size=l))
            read_codes = np.concatenate(out) if out else np.zeros(0, np.uint8)
            for k in mm:
                if k < read_codes.shape[0]:
                    read_codes[k] = rng.choice(BASES[BASES != read_codes[k]])
        read_codes = np.asarray(read_codes, np.uint8)
        lq = int(read_codes.shape[0]) if l_qseq is None else l_qseq
        if qual is None:
            qual = rng.choice(np.array([40, 37, 30, 22, 20, 12, 2], np.uint8), size=lq)
        self.recs.append(dict(pos=int(pos), ops=ops, codes=read_codes, flag=flag, mapq=mapq, lib=lib, nm=nm, sm=sm,
                              qual=np.asarray(qual, np.uint8), lead=lead, l_qseq=lq))

    def build(self):
        assert all(a["pos"] <= b["pos"] for a, b in zip(self.recs, self.recs[1:])), "reads out of position order"
        bb = BatchBuilder()
        qlen = 0
        for k, r in enumerate(self.recs):
            q = r["qual"]
            nxt = self.recs[k + 1]["lead"] if k + 1 < len(self.recs) else None
            want = int(self.rng.integers(0, 4)) if nxt is None else nxt
            pad = (want - (qlen + q.shape[0])) % 4
            q = np.concatenate([q, self.rng.choice(PAD_BYTES, size=pad)]).astype(np.uint8)
            qlen += q.shape[0]
            c = r["codes"]
            if c.shape[0] & 1:
                c = np.concatenate([c, [int(self.rng.integers(0, 16))]])
            seq4 = ((c[0::2] << 4) | c[1::2]).astype(np.uint8)
            seq4 = np.concatenate([seq4, self.rng.integers(0, 256, size=int(self.rng.integers(0, 3))).astype(np.uint8)])
            bb.add(tid=0, pos=r["pos"], flag=r["flag"], mapq=r["mapq"], lib=r["lib"], cigar=[(l << 4) | o for l, o in r["ops"]],
                   seq4=seq4, qual=q, nm=r["nm"], sm=r["sm"], l_qseq=r["l_qseq"], qname=f"k{k}")
        return bb.build()


def _phases(B, p0):
    """64 phase pairs x both strands, M lengths 1-49, mismatches at every lane, runs across steps and across ops."""
    rng = B.rng
    idx = 0
    for rep in range(3):
        for a in range(8):
            for b in range(8):
                m = 1 + (idx * 7 + rep) % 49
                lane = idx % 16
                mm = {j for j in range(m) if j % 16 == lane}
                if m > 17:
                    mm |= {15, 16}
                if m > 34:
                    mm |= {31, 32, 33}
                mm |= {j for j in range(m) if rng.random() < 0.08}
                gap = ("", "D", "N", "I")[idx % 4]
                m2 = 1 + (idx * 5) % 40
                # read nibble phase at the first M op: (2 * seq_off + soft clip) mod 8, the pool offset being unknown here: the
                # clip cycles through 0-7 and the audit checks which phases were reached
                s = (a + 3 * rep) % 8
                cig = (f"{s}S" if s else "") + f"{m}M" + (f"{1 + idx % 5}{gap}{m2}M" if gap else "")
                mm2 = set()
                if gap:
                    mm |= {m - 1}
                    ins = 1 + idx % 5 if gap == "I" else 0
                    mm2 = {m + ins, m + ins + 1} | {m + ins + j for j in range(m2) if rng.random() < 0.1}
                pos = p0 + 8 * idx + b
                B.add(pos, cig, mm=sorted(j + s for j in mm) + sorted(j + s for j in mm2), flag=16 * (idx & 1), lead=idx % 4)
                idx += 1
    return p0 + 8 * idx + 64


def _codes(B, p0):
    """Every (read code, reference code) pair, each reference code spelled two ways."""
    for v, chars in enumerate(CODE_CHARS):
        base = p0 + v * 400
        seg = np.frombuffer(chars * 16, np.uint8)
        B.ref[base:base + 256] = seg
        for k in range(16):
            p = np.arange(256)
            B.add(base, "256M", read_codes=((p // 16 + k) % 16).astype(np.uint8), flag=16 * (k & 1), lead=k % 4, nm=k)
    return p0 + 1000


def _quals(B, p0):
    rng = B.rng
    pos = p0
    k = 0
    lengths = list(range(1, 13)) + [150, 151]
    # every byte value stops the scan of some read, on both strands and at every lead
    for v in range(256):
        for rev in (0, 16):
            lq = lengths[k % len(lengths)]
            run = int(rng.integers(0, lq))                 # Q2 bytes at the 3' end before the byte that stops the scan
            q = rng.choice(np.array([40, 30, 20, 2, 0x82], np.uint8), size=lq)
            if rev:
                q[:run] = 2; q[run] = v
            else:
                q[lq - run:] = 2; q[lq - 1 - run] = v
            B.add(pos, f"{lq}M", mm=[j for j in range(lq) if rng.random() < 0.1], flag=rev, qual=q, lead=k % 4, lib=k % 3)
            k += 1; pos += 1
    # Q2 runs of every length, up to the whole read, with soft clips at both ends: each clamp of three_prime_index binds
    for lq in lengths:
        for run in sorted({0, 1, 2, lq // 3, lq // 2, lq - 1, lq}):
            for rev in (0, 16):
                for lc, rc in ((0, 0), (min(2, lq - 1), 0), (0, min(3, lq - 1)), (min(lq // 3, 30), min(lq // 4, 30))):
                    m = lq - lc - rc
                    if m < 1:
                        continue
                    q = rng.choice(np.array([40, 30, 20], np.uint8), size=lq)
                    if rev:
                        q[:run] = 2
                    else:
                        q[lq - run:] = 2
                    cig = (f"{lc}S" if lc else "") + f"{m}M" + (f"{rc}S" if rc else "")
                    B.add(pos, cig, flag=rev, qual=q, lead=k % 4)
                    k += 1; pos += 1
    # H before S (the S counts as a right clip, R:bamreadcount.cpp:187-192), = / X, P, H, op 9, no CIGAR
    shapes = ["3H4S20M", "2H5S30M3S", "1H6S10M2H", "10=2X8=", "20X", "12=", "5M2P3I10M", "3H20M2H", "10M1B10M", "4S10=3S",
              "8M2D8=1X", "6M1I1P6M"]
    for rep in range(8):
        for sh in shapes:
            lq = sum(l for l, o in ((int(c) >> 4, int(c) & 15) for c in parse_cigar_string(sh)) if o in (0, 1, 4, 7, 8))
            q = rng.choice(np.array([40, 30, 2], np.uint8), size=lq)
            B.add(pos, sh, mm=[j for j in range(lq) if rng.random() < 0.2], flag=16 * (rep & 1), qual=q, lead=rep % 4)
            pos += 1
        B.add(pos, [], read_codes=rng.choice(BASES, size=9), flag=16 * (rep & 1), lead=(rep + 1) % 4)   # mapped, no CIGAR
        pos += 1
    # flags, tags and libraries (and placed unmapped reads when the case keeps them: drawn either way, so that every other
    # read is the same in both forms of the case)
    tags = [dict(nm=None), dict(flag=3, sm=17), dict(flag=3, sm=None), dict(flag=3, sm=-5), dict(flag=2 | 16, sm=0),
            dict(mapq=19), dict(mapq=20), dict(mapq=21), dict(mapq=0), dict(mapq=255), dict(flag=256), dict(flag=512),
            dict(flag=1024), dict(flag=4), dict(lib=None), dict(lib=1), dict(lib=2), dict(nm=-3), dict(nm=0)]
    for rep in range(4):
        for t in tags:
            kw = dict(t)
            B.add(pos, "30M", mm=[3, 4, 20], lead=rep % 4, **kw)
            if kw.get("flag") == 4 and not B.unmapped:
                B.recs.pop()
            pos += 1
    return pos + 200


def _sparse(B, p0):
    rng = B.rng
    for k in range(128):                                    # first positions 80 apart: 10,160 bases > 2 * K0_REF_CAP
        B.add(p0 + 80 * k, "60M", mm=[k % 60, (k + 1) % 60], flag=16 * (k & 1), lead=k % 4)
    p = p0 + 80 * 128 + 100
    for k in range(384):                                    # dense blocks, every 24th read jumping past the staged window
        if k % 24 == 23:
            B.add(p + 2 * k, f"20M{2500 + 100 * (k % 5)}{'DN'[k & 1]}25M", mm=[19, 20, 21, 44], flag=16 * (k & 1), lead=k % 4)
        else:
            B.add(p + 2 * k, "50M", mm=[int(rng.integers(0, 50))], lead=k % 4)
    return p + 768 + 8000


def _long(B, p0):
    rng = B.rng
    pos = p0
    special = ["2048M", "2049M", "1S2048M", "1S2049M", "2048M1S", "2S2047M", "2050M"]
    for k in range(224):
        if k < len(special):
            cig = special[k]
        else:
            m = int(rng.integers(200, 1800))
            s = k % 8
            # four M ops, each starting at another nibble phase of the read and of the reference
            q4 = m // 8
            cig = ((f"{s}S" if s else "") + f"{m // 2}M{1 + k % 3}{'DNI'[k % 3]}{q4}M{1 + (k // 3) % 4}{'IDN'[k % 3]}{q4}M"
                   f"{2 + k % 5}{'NID'[k % 3]}{m - m // 2 - 2 * q4}M" + ("7S" if k % 5 == 0 else ""))
        lq = sum(l for l, o in ((int(c) >> 4, int(c) & 15) for c in parse_cigar_string(cig)) if o in (0, 1, 4, 7, 8))
        q = rng.choice(np.array([40, 30, 20], np.uint8), size=lq)
        if k % 3 == 0 or k % 16 in (7, 8, 9, 10, 11, 13):
            run = lq - (k % 16 == 9) if k % 16 in (7, 8, 9, 10, 11, 13) else int(rng.integers(0, lq))
            if k & 1:
                q[:run] = 2
            else:
                q[lq - run:] = 2
        mm = {int(x) for x in rng.integers(0, lq, size=lq // 25)} | {15, 16, 17}
        if k >= len(special):                               # a mismatch at each side of the op between the two M ops
            mm |= {s + m // 2 - 1, s + m // 2 + (1 + k % 3 if k % 3 == 2 else 0)}
        B.add(pos + int(rng.integers(0, 8)), cig, mm=sorted(mm), flag=16 * (k & 1), qual=q, lead=(k + k // 8) % 4, nm=int(rng.integers(0, 9)))
        pos += 40
    # more than 65,535 CIGAR ops
    n_ops = 33_000
    B.add(pos, [(1 << 4) | 0, (1 << 4) | 2] * n_ops, mm=[5, 6, 7, 1000], lead=1)
    return pos + 2 * n_ops + 100


def _ends(B, p0):
    """Reads running off the supplied window, and past chrom_len (the window does not reach it)."""
    rng = B.rng
    for k in range(40):                                     # M ops running past the end of the supplied window
        p = WIN_END - 60 + k
        B.add(p, f"{70 + k % 9}M", mm=[1, 2, 50, 60, 69], flag=16 * (k & 1), lead=k % 4)
    p = WIN_END - 20
    L = CHROM_LEN
    gap = L - p
    for k, cig in enumerate([f"10M{gap - 17}N20M4S",          # second M op straddles chrom_len: the walk stops at the NUL
                             f"10M{gap - 10}D10M3S",          # second M op starts exactly at chrom_len
                             f"10M{gap - 7}N10M5S",           # ... three past it: -l skips its positions and walks on
                             f"10M{gap - 11}D1M1D6M2S",       # one ending at it, then one past it
                             f"4S6M{gap - 6}N12M"]):
        for rev in (0, 16):
            B.add(p, cig, mm=[4, 5], flag=rev, lead=(k + rev) % 4)
    return L


@functools.lru_cache(maxsize=None)
def k0_case(seed=911, unmapped=False):
    """The case.  A push never admits a placed unmapped read, and one in the batch keeps brc_push_reads from borrowing it,
    so the pushed form has none and goes down the pipelined path on its own pools; unmapped=True adds four, for
    brc_run_device, which hands K0 every read it is given."""
    B = _Builder(seed, unmapped)
    p = WIN_BEG + 100
    for section in (_phases, _codes, _quals, _sparse, _long):
        p = section(B, p)
    assert p < WIN_END - 100, p
    _ends(B, p)
    batch = B.build()
    ref = B.ref
    return dict(name="k0_unmapped" if unmapped else "k0", contigs=[("k0", CHROM_LEN, ref[WIN_BEG:WIN_END].tobytes(), WIN_BEG)], batch=batch,
                regions=[(0, WIN_BEG + 2, WIN_END)], site_list=False, modes=(False, True), lib_names=["lib0", "lib1", "lib2"])
