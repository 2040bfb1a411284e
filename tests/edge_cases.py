"""Hand-built / fuzzed edge-case reads the reference's own fixtures never exercise
(SURVEY.md §4 "What nothing covers"): D / N / = / X / H / P ops, several indel alleles at one
site, IUPAC and lower-case reference bases, missing NM / SM tags, filtered flags, reads without a
library under -p, all-Q2 reads, a read overhanging the contig end, adjacent argv regions (the
never-cleared deletion queue, SURVEY.md A.6).  Deterministic (seeded)."""
from __future__ import annotations

import numpy as np

from bam_readcount_b200.batch import BatchBuilder

_OPS = "MIDNSHP=XB"


def _rand_cigar(rng, target_q):
    """Random valid CIGAR consuming exactly target_q query bases. Returns (ops list[(len,op)], ref_span)."""
    ops = []
    q_left = target_q
    if rng.random() < 0.15:
        ops.append((int(rng.integers(1, 6)), "H"))
    if rng.random() < 0.3 and q_left > 12:
        s = int(rng.integers(1, 8)); ops.append((s, "S")); q_left -= s
    tail_s = 0
    if rng.random() < 0.3 and q_left > 12:
        tail_s = int(rng.integers(1, 8)); q_left -= tail_s
    n_blocks = int(rng.integers(1, 5))
    if rng.random() < 0.08:            # read whose first reference-consuming op is a deletion
        ops.append((int(rng.integers(1, 4)), "D"))
    for b in range(n_blocks):
        last = b == n_blocks - 1
        m = q_left if last else int(rng.integers(1, max(2, q_left - 3 * (n_blocks - b))))
        m = max(1, min(m, q_left))
        ops.append((m, rng.choice(["M", "M", "M", "=", "X"])))
        q_left -= m
        if last or q_left <= 2:
            if q_left > 0:
                ops.append((q_left, "M")); q_left = 0
            break
        r = rng.random()
        if r < 0.3:
            i = int(rng.integers(1, min(4, q_left))); ops.append((i, "I")); q_left -= i
        elif r < 0.55:
            ops.append((int(rng.integers(1, 5)), "D"))
        elif r < 0.65:
            ops.append((int(rng.integers(1, 30)), "N"))
        elif r < 0.75:
            i = int(rng.integers(1, min(3, q_left))); ops.append((int(rng.integers(1, 3)), "P")); ops.append((i, "I")); q_left -= i
        elif r < 0.85:
            i = int(rng.integers(1, min(3, q_left))); ops.append((i, "I")); q_left -= i; ops.append((int(rng.integers(1, 4)), "D"))
        else:
            ops.append((int(rng.integers(1, 4)), "D"))
            if q_left > 2:
                i = int(rng.integers(1, min(3, q_left))); ops.append((i, "I")); q_left -= i
        if q_left <= 0:   # must end on a match-type op
            last_len, last_op = ops[-1]
            # steal one base from the previous match block
            for k in range(len(ops) - 1, -1, -1):
                if ops[k][1] in "M=X" and ops[k][0] > 1:
                    ops[k] = (ops[k][0] - 1, ops[k][1]); q_left += 1; break
            ops.append((max(q_left, 1), "M")); q_left = 0
            break
    if tail_s:
        ops.append((tail_s, "S"))
    if rng.random() < 0.1:
        ops.append((int(rng.integers(1, 6)), "H"))
    # merge accidental adjacent identical ops
    merged = []
    for l, o in ops:
        if merged and merged[-1][1] == o:
            merged[-1] = (merged[-1][0] + l, o)
        else:
            merged.append((l, o))
    ops = merged
    q = sum(l for l, o in ops if o in "MIS=X")
    assert q == target_q, (ops, q, target_q)
    span = sum(l for l, o in ops if o in "MDN=X")
    return ops, span


def _ref(rng, L, messy=True):
    r = rng.choice(list(b"ACGT"), size=L).astype(np.uint8)
    if messy:
        for ch, p in ((ord("N"), 0.02), (ord("a"), 0.02), (ord("g"), 0.02), (ord("R"), 0.01), (ord("y"), 0.01), (ord("n"), 0.005)):
            r[rng.random(L) < p] = ch
    return r


def _read_from_ref(rng, ref, pos, ops, sub_rate=0.06):
    """Build the query bases for a CIGAR so most match positions agree with the reference."""
    q = []
    rp = pos
    for l, o in ops:
        if o in "M=X":
            for j in range(l):
                c = chr(ref[rp + j]).upper() if rp + j < len(ref) else "A"
                if c not in "ACGT":
                    c = "ACGT"[int(rng.integers(0, 4))]
                if rng.random() < sub_rate:
                    c = rng.choice(["A", "C", "G", "T", "N", "R"], p=[0.22, 0.22, 0.22, 0.22, 0.08, 0.04])
                q.append(c)
            rp += l
        elif o in "DN":
            rp += l
        elif o in "IS":
            for _ in range(l):
                q.append(rng.choice(["A", "C", "G", "T", "N", "M"], p=[0.24, 0.24, 0.24, 0.24, 0.03, 0.01]))
    return "".join(q)


def _quals(rng, n, reverse):
    q = rng.choice([40, 37, 30, 25, 20, 19, 12, 2], size=n).astype(np.uint8)
    r = rng.random()
    if r < 0.25:      # Q2 run at the 3' end (forward: tail; reverse: head)
        t = int(rng.integers(1, max(2, n // 2)))
        if reverse:
            q[:t] = 2
        else:
            q[n - t:] = 2
    elif r < 0.30:
        q[:] = 2       # every base Q2
    elif r < 0.35:     # Q2 run at the wrong end
        t = int(rng.integers(1, 5))
        if reverse:
            q[n - t:] = 2
        else:
            q[:t] = 2
    return q


def fuzz_case(seed=3, L=400, n_reads=220, name="fuzz", per_lib_safe=False, n_libs=3, overhang=True, force_perlib=False):
    rng = np.random.default_rng(seed)
    ref = _ref(rng, L)
    bb = BatchBuilder()
    starts = np.sort(rng.integers(5, L - 90, size=n_reads))
    recs = []
    for i, p in enumerate(starts):
        lq = int(rng.integers(20, 70))
        ops, span = _rand_cigar(rng, lq)
        if p + span >= L - 2:
            continue
        flag = 0
        if rng.random() < 0.5:
            flag |= 16
        sm = None
        if rng.random() < 0.4:
            flag |= 1 | 2
            if rng.random() < 0.6:
                sm = int(rng.integers(0, 61))
        r = rng.random()
        if r < 0.04:
            flag |= 256
        elif r < 0.08:
            flag |= 512
        elif r < 0.12:
            flag |= 1024
        elif r < 0.15:
            flag |= 4
        seq = _read_from_ref(rng, ref, int(p), ops)
        nm = None if rng.random() < 0.1 else int(rng.integers(0, 6))
        lib = int(rng.integers(0, n_libs))
        if not per_lib_safe and rng.random() < 0.05:
            lib = None
        recs.append(dict(tid=0, pos=int(p), flag=flag, mapq=int(rng.choice([60, 60, 40, 29, 20, 19, 0])), lib=lib,
                         cigar="".join(f"{l}{o}" for l, o in ops), seq=seq, qual=_quals(rng, lq, bool(flag & 16)), nm=nm, sm=sm,
                         qname=f"f{i}"))
    if overhang:   # a read running past the contig end: the reference walk stops at ref[len]==0 (R:...:151)
        lq = 30
        recs.append(dict(tid=0, pos=L - 12, flag=0, mapq=60, lib=0, cigar="30M", seq="ACGT" * 7 + "AC", qual=np.full(lq, 35, np.uint8),
                         nm=1, sm=None, qname="overhang"))
    recs.sort(key=lambda r: r["pos"])
    for r in recs:
        bb.add_sam(**r)
    batch = bb.build()
    fs = {"default": dict(), "q20b20": dict(min_mapq=20, min_bq=20), "ic": dict(insertion_centric=True), "d3": dict(max_cnt=3)}
    if per_lib_safe or force_perlib:
        fs["perlib"] = dict(per_lib=True)
        fs["perlib_ic_q20"] = dict(per_lib=True, insertion_centric=True, min_mapq=20)
    return dict(name=name, contigs=[("c", L, ref.tobytes(), 0)], batch=batch, regions=[(0, 1, L)], site_list=True,
                lib_names=[f"lib{i}" for i in range(n_libs)], flag_sets=fs)


def multi_allele_case(seed=9, L=300, name="alleles"):
    """Many reads over one window: several insertion alleles (same and different lengths, IUPAC bases
    that canonicalise to N) and several deletion lengths anchored at the same site."""
    rng = np.random.default_rng(seed)
    ref = _ref(rng, L, messy=False)
    ref[150:160] = np.frombuffer(b"acgtNNacgt", dtype=np.uint8)   # deletion alleles keep FASTA case
    bb = BatchBuilder()
    recs = []
    ins_alleles = ["A", "C", "AC", "AG", "R", "M", "ACGTACGTACGTACGTACGTACGTACGTACGTACGTA", "N"]
    for i in range(160):
        p = int(rng.integers(100, 140))
        anchor = 149 - p + 1            # match length before the indel so that it sits after reference pos 148/149
        anchor = max(3, anchor - int(rng.integers(0, 2)))
        kind = rng.random()
        if kind < 0.35:
            a = ins_alleles[int(rng.integers(0, len(ins_alleles)))]
            tailm = 25
            cigar = f"{anchor}M{len(a)}I{tailm}M"
            body = _read_from_ref(rng, ref, p, [(anchor, "M")], 0.02) + a + _read_from_ref(rng, ref, p + anchor, [(tailm, "M")], 0.02)
        elif kind < 0.7:
            dl = int(rng.choice([1, 2, 3, 7]))
            tailm = 25
            cigar = f"{anchor}M{dl}D{tailm}M"
            body = _read_from_ref(rng, ref, p, [(anchor, "M")], 0.02) + _read_from_ref(rng, ref, p + anchor + dl, [(tailm, "M")], 0.02)
        else:
            tailm = 30
            cigar = f"{anchor + tailm}M"
            body = _read_from_ref(rng, ref, p, [(anchor + tailm, "M")], 0.03)
        flag = 16 if rng.random() < 0.5 else 0
        recs.append(dict(tid=0, pos=p, flag=flag, mapq=int(rng.choice([60, 50, 30, 10])), lib=int(rng.integers(0, 2)), cigar=cigar,
                         seq=body, qual=_quals(rng, len(body), bool(flag)), nm=int(rng.integers(0, 4)), sm=None, qname=f"a{i}"))
    recs.sort(key=lambda r: r["pos"])
    for r in recs:
        bb.add_sam(**r)
    return dict(name=name, contigs=[("c", L, ref.tobytes(), 0)], batch=bb.build(),
                # argv regions, the last three adjacent: exercises the never-cleared deletion queue
                regions=[(0, 100, 200), (0, 148, 148), (0, 149, 149), (0, 150, 150), (0, 151, 152)], site_list=False,
                lib_names=["lib0", "lib1"],
                flag_sets={"default": dict(), "ic": dict(insertion_centric=True), "perlib": dict(per_lib=True),
                           "q20b20": dict(min_mapq=20, min_bq=20)})


def all_cases():
    return [fuzz_case(3, name="fuzz_a"), fuzz_case(17, L=500, n_reads=400, name="fuzz_b"),
            fuzz_case(23, name="fuzz_plib", per_lib_safe=True), fuzz_case(29, name="fuzz_nolib", per_lib_safe=False, overhang=False, force_perlib=True),
            multi_allele_case()]


# the fresh-fuzz seeds: cases of their own, not the ones above (tests/test_differential_fuzz.py, make_golden.py)
FRESH_SEEDS = (101, 102, 103, 104, 105, 106)


def fresh_fuzz_case(seed):
    rng = np.random.default_rng(seed)
    safe = bool(seed % 2)
    return fuzz_case(seed, L=int(rng.integers(300, 700)), n_reads=int(rng.integers(150, 380)), name=f"fresh{seed}",
                     per_lib_safe=safe, n_libs=int(rng.integers(1, 6)), overhang=bool(seed % 3), force_perlib=not safe)
