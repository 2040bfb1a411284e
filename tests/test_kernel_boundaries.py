"""The kernels at their capacity limits (tests/boundary_cases.py), bit for bit.

CPU
  audit   the capacities are parsed out of csrc/; from each case's batch the test recomputes what the kernels will decide (K0's
          staged blocks and reference window, the producer's chunk cuts and CIGAR staging, FM_FASTDIV / FM_HOT per read, per-site
          depth and 16-bit sums, deep-tile read counts) and asserts that every target of the case lands on both sides of its
          limit.  If a constant changes, the failing target names the case that no longer straddles it.
  anchor  the oracle's text on every case and flag set against the SHA-256 of what the unmodified reference binary printed
          (tests/golden/boundary_sha256.json, written by tests/golden/make_golden.py).
GPU
  the engine against the oracle on every case and flag set (raw accumulators, text, warning counters), forced through the
  deep-site kernel, as one borrowed push and as two pushes; the reciprocal-division self-test over every hot-path numerator;
  secondary-pool growth; the site selection at scale."""
import functools
import hashlib
import json
import os
import re

import numpy as np
import pytest

import boundary_cases
import cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bam_readcount_b200", "csrc")
GOLDEN = os.path.join(ROOT, "tests", "golden")

_CONST_NAMES = ("TILE", "STAGE_READS", "STAGE_QUAL", "STAGE_SEQ", "STAGE_CIGAR", "K0_READS", "K0_QUAL_CAP", "K0_SEQ_CAP", "K0_REF_CAP",
                "FASTDIV_MAX", "DEEP_THREADS", "DEEP_ICACHE", "SEL_LAST_ROWS", "SCAN_CTA")


@functools.lru_cache(maxsize=None)
def kernel_constants():
    """constexpr int NAME = <expression over earlier names>; from csrc/ (BRC_STAGE_READS from its #define)."""
    src = "".join(open(os.path.join(CSRC, f)).read() for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh", ".h")))
    env = {}
    m = re.search(r"#define\s+BRC_STAGE_READS\s+(\d+)", src)
    env["BRC_STAGE_READS"] = int(m.group(1))
    for name in _CONST_NAMES:
        m = re.search(r"constexpr\s+int\s+" + name + r"\s*=\s*([^;]+);", src)
        assert m, f"{name} not found in csrc/"
        env[name] = int(eval(m.group(1), {}, dict(env)))
    return env


def _first_diff(a: str, b: str) -> str:
    la, lb = a.splitlines(), b.splitlines()
    for i, (x, y) in enumerate(zip(la, lb)):
        if x != y:
            return f"line {i}:\n got: {x[:300]}\nwant: {y[:300]}"
    return f"length differs: got {len(la)} lines, want {len(lb)}"


# ---------------------------------------------------------------------------------------------------------------------------
# what the kernels decide, recomputed on the host
# ---------------------------------------------------------------------------------------------------------------------------
def _reads_view(b):
    """Per read: list of (len, op char) and the decoded quality / base arrays."""
    ops = "MIDNSHP=XB"
    co = b.cigar_off.astype(np.int64)
    out = []
    for i in range(b.n_reads):
        out.append([(int(c) >> 4, ops[int(c) & 15]) for c in b.cigar[co[i]:co[i + 1]]])
    return out


def read_facts(case, batch, site_list):
    """fetch_func's per-read values as K0 forms them (brc_kernels.cu read_precompute_kernel)."""
    K = kernel_constants()
    name, clen_chrom, seq, wb = case["contigs"][0]
    ref = np.frombuffer(case.get("full_ref", seq), np.uint8)
    from bam_readcount_b200.batch import _NT16
    refc = _NT16[ref]
    cig = _reads_view(batch)
    so = batch.seq_off.astype(np.int64)
    qo = batch.qual_off.astype(np.int64)
    facts = []
    for i, ops in enumerate(cig):
        lq = int(batch.l_qseq[i])
        pk = batch.seq[so[i]:so[i + 1]]
        nib = np.empty(pk.shape[0] * 2, np.uint8); nib[0::2] = pk >> 4; nib[1::2] = pk & 15
        qual = batch.qual[qo[i]:qo[i + 1]]
        refops = [o for _, o in ops if o in "MDN=X"]
        simple = len(refops) == 1 and refops[0] in "M=X" and not any(o in "IP" for _, o in ops)
        lclip, clen = 0, lq
        refpos, rp, walking = int(batch.pos[i]), 0, True
        mm = []                       # (read offset, quality) of mismatches
        for k, (l, o) in enumerate(ops):
            if not walking:
                break
            if o == "M":
                jn, hit = l, False
                if refpos + l > clen_chrom:
                    if site_list and refpos > clen_chrom:
                        jn = 0
                    else:
                        jn, hit = max(0, clen_chrom - refpos), True
                for j in range(jn):
                    r, q = int(refc[refpos + j]), int(nib[rp + j])
                    if r != q and r != 15 and q != 0:
                        mm.append((rp + j, int(qual[rp + j])))
                if hit:
                    walking = False
                else:
                    refpos += l; rp += l
            elif o in "DN":
                refpos += l
            elif o == "I":
                rp += l
            elif o == "S":
                rp += l; clen -= l
                if k == 0:
                    lclip += l
        mmq, last_p, last_q = 0, -1, 0
        for p, q in mm:
            if last_p != -1 and last_p + 1 != p:
                mmq += last_q; last_q = q
            elif last_p != -1:
                last_q = max(last_q, q)
            else:
                last_q = q
            last_p = p
        mmq += last_q
        fast = 1 <= lq <= K["FASTDIV_MAX"] and 1 <= clen <= K["FASTDIV_MAX"]
        nm_ok = int(batch.nm[i]) != -2 ** 31
        sm_missing = bool(batch.flag[i] & 2) and int(batch.sm[i]) == -2 ** 31
        qoff = 0
        for l, o in ops:
            if o in "MDN=X":
                break
            if o == "S":
                qoff += l
        se = (int(batch.sm[i]) if not sm_missing else 0) if batch.flag[i] & 2 else int(batch.mapq[i])
        facts.append(dict(lq=lq, clen=clen, lclip=lclip, fast=fast, hot=simple and fast and nm_ok and not sm_missing, simple=simple,
                          qoff=qoff, mmq=mmq, se=se, ops=ops))
    return facts


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


def site_sums(batch, facts, lo, hi):
    """Per site in [lo, hi): depth, and the clipped-length / SE / mismatch-quality sums over covering live reads (every event of
    the stacks that target the 16-bit sums passes and lands in the primary class)."""
    n = hi - lo
    depth = np.zeros(n + 1, np.int64); clip = np.zeros(n + 1, np.int64); se = np.zeros(n + 1, np.int64); mmq = np.zeros(n + 1, np.int64)
    e = batch.ref_end()
    for i, f in enumerate(facts):
        a, b = max(int(batch.pos[i]), lo) - lo, min(int(e[i]), hi) - lo
        if b <= a:
            continue
        depth[a] += 1; depth[b] -= 1
        if batch.flag[i] & 1024:
            continue
        clip[a] += f["clen"]; clip[b] -= f["clen"]
        se[a] += f["se"] & 0xFFFFFFFF; se[b] -= f["se"] & 0xFFFFFFFF
        mmq[a] += f["mmq"]; mmq[b] -= f["mmq"]
    return {k: np.cumsum(v)[:n] for k, v in (("depth", depth), ("clip", clip), ("se", se), ("mmq", mmq))}


def _both(lo_side, hi_side, what):
    assert lo_side and hi_side, f"{what}: below the limit {'hit' if lo_side else 'MISSED'}, above it {'hit' if hi_side else 'MISSED'}"


def check_targets(case):
    K = kernel_constants()
    T = K["TILE"]
    ci, b1, e1 = case["regions"][0]
    tid, beg, end, batch = cases.region_reads(case, ci, b1, e1)
    if batch.n_reads != case["batch"].n_reads:      # site-list cases: per-read facts over every read of the case
        batch = case["batch"]
    facts = read_facts(case, batch, case["site_list"])
    first_pos = max(beg, 0)
    for target in case["targets"]:
        if target == "k0_qual_cap":
            bl = [b for b in k0_blocks(batch, case) if b["uniform"]]
            _both(any(b["staged"] and b["lq"] * K["K0_READS"] + 32 > K["K0_QUAL_CAP"] - 160 for b in bl),
                  any(not b["staged"] and b["lq"] * K["K0_READS"] <= K["K0_QUAL_CAP"] + 160 for b in bl), target)
        elif target == "k1_stage_shrink":
            ch = [c for c in k1_chunks(batch, tile_ranges(batch, first_pos, end)) if c["full"] == K["STAGE_READS"] and len(c["lq"]) == 1]
            _both(any(c["r1"] - c["r0"] == c["full"] and c["staged"] and max(c["lq"]) * K["STAGE_READS"] + 32 == K["STAGE_QUAL"] for c in ch),
                  any(c["r1"] - c["r0"] < c["full"] and c["staged"] and max(c["lq"]) * K["STAGE_READS"] + 32 == K["STAGE_QUAL"] + K["STAGE_READS"]
                      for c in ch), target)
        elif target == "fastdiv_len":
            M = K["FASTDIV_MAX"]
            _both(any(f["lq"] == M and f["fast"] for f in facts), any(f["lq"] == M + 1 and not f["fast"] for f in facts), target)
        elif target == "fastdiv_clen":
            M = K["FASTDIV_MAX"]
            _both(any(f["clen"] == M and f["lq"] > M and not f["fast"] for f in facts) and any(f["clen"] == M and f["fast"] for f in facts),
                  any(f["clen"] == M + 1 and not f["fast"] for f in facts), target)
        elif target == "fastdiv_numerator":
            # largest |2 (qpos - left_clip) - clipped_length| of a hot read against the bound 2 b + 2 the self-test once stopped at:
            # the controls (soft clip first, or clips only at the end) stay inside it; nH mS kM reads on both strands go far past it
            def num(f):
                return max(abs(2 * (f["qoff"] - f["lclip"]) - f["clen"]), abs(2 * (f["qoff"] + f["clen"] - 1 - f["lclip"]) - f["clen"]))
            hot = [(i, f) for i, f in enumerate(facts) if f["hot"]]
            ctrl = [f for _, f in hot if f["ops"][0][1] != "H"]
            hs = [(i, f) for i, f in hot if f["ops"][0][1] == "H" and f["qoff"] > 0]
            _both(any(f["ops"][0][1] == "S" for f in ctrl) and any(f["ops"][0][1] == "M" for f in ctrl)
                  and all(num(f) <= 2 * f["clen"] + 2 for f in ctrl),
                  {int(batch.flag[i]) & 16 for i, _ in hs} == {0, 16} and all(num(f) > 2 * f["clen"] + 2 for _, f in hs)
                  and max(num(f) for _, f in hs) > 2 * K["FASTDIV_MAX"] - 100, target)
        elif target == "k0_ref_window":
            bl = k0_blocks(batch, case)
            _both(any(b["staged"] and b["ref_staged"] for b in bl),
                  any(b["ref_staged"] and b["past"] for b in bl) and any(b["staged"] and not b["ref_staged"] and b["span"] > 2 * K["K0_REF_CAP"]
                                                                          for b in bl), target)
        elif target == "chunk_reads":
            sizes = [h - l for l, h in tile_ranges(batch, first_pos, end)]
            S = K["STAGE_READS"]
            _both(S in sizes, S + 1 in sizes and 2 * S in sizes, target)
        elif target == "hot_run_end":
            ch = k1_chunks(batch, tile_ranges(batch, first_pos, end))
            full = [c for c in ch if c["r1"] - c["r0"] == K["STAGE_READS"]]

            def run_len(c):
                n = 0
                for i in range(c["r1"] - 1, c["r0"] - 1, -1):
                    if not facts[i]["hot"]:
                        break
                    n += 1
                return n
            _both(any(run_len(c) % 2 == 1 for c in full), any(run_len(c) % 2 == 0 and run_len(c) > 0 for c in full), target)
        elif target == "warp_edges":
            # in the tile built for it: reads starting at wfirst+31 / wfirst+32 and ending at wfirst / wfirst+1 of each probed warp
            pr = case["probe"]
            starts, ends = set(batch.pos.tolist()), set(batch.ref_end().tolist())
            wfs = [first_pos + pr["warp_tile"] * T + 32 * w for w in pr["warp_windows"]]
            _both(all(wf + 31 in starts and wf in ends for wf in wfs), all(wf + 32 in starts and wf + 1 in ends for wf in wfs), target)
        elif target == "tile_edges":
            starts = set(batch.pos.tolist())
            t0s = [first_pos + t * T for t in case["probe"]["edge_tiles"]]
            _both(all(t0 - 1 in starts for t0 in t0s), all(t0 in starts for t0 in t0s), target)
        elif target == "lead_skip":
            # the tile built for it: more than one ballot (32) of leading reads that end before its last warp's window, then reads
            # that cover that window
            t = case["probe"]["lead_tile"]
            l, h = tile_ranges(batch, first_pos, end)[t]
            last_w = first_pos + t * T + T - 32
            e_ = batch.ref_end()
            lead = 0
            while l + lead < h and e_[l + lead] <= last_w:
                lead += 1
            _both(any(e_[i] > last_w for i in range(l + lead, h)), lead > 32, target)
        elif target == "libless_hot":
            # the tile built for it: hot pairs of reads with a library (the pair body under -p), and a library-less read between two
            # such hot reads (never part of a pair)
            l, h = tile_ranges(batch, first_pos, end)[case["probe"]["libless_tile"]]
            has = lambda i: facts[i]["hot"] and batch.lib[i] != 0xFFFF
            _both(any(has(i) and has(i + 1) for i in range(l, h - 1)),
                  any(batch.lib[i] == 0xFFFF and has(i - 1) and has(i + 1) for i in range(l + 1, h - 1)), target)
        elif target == "queue_rows":
            # an argv region's last site whose covering reads all sit in library rows >= SEL_LAST_ROWS, with a deletion anchored
            # there, and a later region holding the next site (where the deletion prints); the same with rows below it
            SL = K["SEL_LAST_ROWS"]
            e_ = batch.ref_end()
            regs = [(b - 1, e - 1) for _, b, e in case["regions"]]

            def anchored(a, rows_ok):
                cov = [i for i in range(batch.n_reads) if batch.pos[i] <= a < e_[i]]
                dels = [i for i in cov if facts[i]["ops"][0][1] == "M" and facts[i]["ops"][1][1] == "D"
                        and batch.pos[i] + facts[i]["ops"][0][0] - 1 == a]
                ends_region = [k for k, (b, e) in enumerate(regs) if e == a]
                later = ends_region and any(b <= a + 1 <= e for b, e in regs[ends_region[0] + 1:])
                return bool(cov) and all(batch.lib[i] != 0xFFFF and rows_ok(int(batch.lib[i])) for i in cov) and bool(dels) and bool(later)
            _both(all(anchored(a, lambda r: r < SL) for a in case["probe"]["low_anchors"]),
                  all(anchored(a, lambda r: r >= SL) for a in case["probe"]["anchors"]) and len(case["lib_names"]) > SL + 4, target)
        elif target == "cigar_stage":
            ch = [c for c in k1_chunks(batch, tile_ranges(batch, first_pos, end)) if c["r1"] - c["r0"] == K["STAGE_READS"]]
            _both(any(c["cstaged"] and c["cops"] > K["STAGE_CIGAR"] - 8 for c in ch),
                  any(not c["cstaged"] and c["cops"] <= K["STAGE_CIGAR"] + 8 for c in ch), target)
        elif target in ("ncover_8bit", "clip_sum_16bit", "se_sum_16bit", "mmq_sum_16bit"):
            s = site_sums(batch, facts, first_pos, end)
            key, lim = {"ncover_8bit": ("depth", 255), "clip_sum_16bit": ("clip", 0xFFFF), "se_sum_16bit": ("se", 0xFFFF),
                        "mmq_sum_16bit": ("mmq", 0xFFFF)}[target]
            v = s[key]
            _both(lim in v and lim - 1 in v if key == "depth" else lim in v, lim + 1 in v, target)
            if key == "se":
                assert (v > 0xFFFFFFFF - 0x10000).any(), "se_sum_16bit: no site whose SE sum wraps below zero"
        elif target == "deep_block":
            counts = []
            for (ci2, b, e) in case["regions"]:
                if e - b + 1 <= 2:
                    _, bg, en, sub = cases.region_reads(case, ci2, b, e)
                    counts.append(sub.n_reads)
            D = K["DEEP_THREADS"]
            _both(D - 1 in counts and D in counts, D + 1 in counts, target)
        elif target == "icache":
            C = K["DEEP_ICACHE"]
            per_site = {}      # distinct short insertion alleles (the inserted nibbles) per anchor site
            so = batch.seq_off.astype(np.int64)
            for i, f in enumerate(facts):
                ops = f["ops"]
                if len(ops) == 3 and ops[1][1] == "I" and ops[1][0] <= 3:
                    pk = batch.seq[so[i]:so[i + 1]]
                    nib = np.empty(pk.shape[0] * 2, np.uint8); nib[0::2] = pk >> 4; nib[1::2] = pk & 15
                    per_site.setdefault(int(batch.pos[i]) + ops[0][0] - 1, set()).add(tuple(nib[ops[0][0]:ops[0][0] + ops[1][0]].tolist()))
            ns = [len(v) for v in per_site.values()]
            _both(C in ns, C + 1 in ns, target)
        elif target == "indel_len":
            ins = {l for f in facts for l, o in f["ops"] if o == "I"}
            dels = {l for f in facts for l, o in f["ops"] if o == "D"}
            _both(8 in ins and 127 in dels, 9 in ins and 128 in dels, target)
        elif target == "byte_values":
            _both(bool((batch.qual == 0xFF).any()), bool((batch.mapq == 255).any()), target)
        else:
            raise AssertionError(f"unknown target {target}")


CASES = boundary_cases.all_cases()


def test_kernel_constants_parse():
    K = kernel_constants()
    assert set(_CONST_NAMES) <= set(K)
    assert K["STAGE_QUAL"] == K["STAGE_READS"] * 152 + 32 and K["K0_QUAL_CAP"] == K["K0_READS"] * 160 + 32


@pytest.mark.parametrize("case", CASES + (boundary_cases.queue_rows(),), ids=[c["name"] for c in CASES] + ["queue_rows"])
def test_case_straddles_its_limits(case):
    check_targets(case)


def test_cases_cover_every_window_start_and_contig_length_residue():
    wins = {c["contigs"][0][3] for c in CASES if c["name"].startswith("refwin")}
    lens = {c["contigs"][0][1] % 4 for c in CASES if c["name"].startswith("refwin")}
    assert wins == {0, 1, 4095, 4097} and lens == {0, 1, 2, 3}
    # reads run to and past the contig end
    for c in CASES:
        if c["name"].startswith("refwin"):
            assert (c["batch"].ref_end() > c["contigs"][0][1]).any()


JOBS = boundary_cases.jobs()


@pytest.mark.parametrize("job", JOBS, ids=[j[4] for j in JOBS])
def test_oracle_equals_reference_binary_on_boundary_cases(job):
    with open(os.path.join(GOLDEN, "boundary_sha256.json")) as fh:
        want = json.load(fh)
    case, fname, fl, sl, key = job
    got, _, _ = cases.run_oracle(case, fl, site_list=sl)
    assert hashlib.sha256(got.encode("latin-1")).hexdigest() == want[key], f"{key}: oracle differs from the reference binary"


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
def _engine_two_pushes(case, flags, site_list):
    """One region, its reads pushed in two halves: the first push is borrowed, then copied when the second arrives."""
    from bam_readcount_b200.engine import Engine
    e = Engine(lib_names=case["lib_names"], **flags)
    try:
        name, clen, seq, wb = case["contigs"][0]
        e.set_reference(0, name, clen, seq, wb)
        ci, b1, e1 = case["regions"][0]
        tid, beg, end, sub = cases.region_reads(case, ci, b1, e1)
        e.begin_region(tid, beg, end, site_list)
        h = sub.n_reads // 2
        e.push_reads(sub.select(np.arange(0, h)))
        e.push_reads(sub.select(np.arange(h, sub.n_reads)))
        e.end_region()
        e.compute()
        return e.format_text(-1), e.warnings()
    finally:
        e.close()


@functools.lru_cache(maxsize=None)
def _oracle(case_name, fname, sl):
    case = {c["name"]: c for c in CASES}[case_name]
    return cases.run_oracle(case, boundary_cases.FLAG_SETS[fname], site_list=sl)


@pytest.mark.gpu
@pytest.mark.parametrize("job", JOBS, ids=[j[4] for j in JOBS])
def test_engine_equals_oracle_on_boundary_cases(job, monkeypatch):
    case, fname, fl, sl, key = job
    otext, odump, owarn = _oracle(case["name"], fname, sl)
    etext, edump, ewarn, _ = cases.run_engine(case, fl, site_list=sl, want_dump=True)
    assert edump == odump, _first_diff(edump, odump)
    assert etext == otext, _first_diff(etext, otext)
    assert (ewarn[0], ewarn[1], ewarn[3]) == owarn
    if len(case["regions"]) == 1 and "max_cnt" not in fl:
        t2, w2 = _engine_two_pushes(case, fl, sl)          # the copy path (run_engine's one push is the pipelined path)
        assert t2 == otext, _first_diff(t2, otext)
        assert (w2[0], w2[1], w2[3]) == owarn
    if sl:
        monkeypatch.setenv("BRC_DEEP_MIN_READS", "1")
        etext, edump, ewarn, _ = cases.run_engine(case, fl, site_list=sl, want_dump=True)
        assert edump == odump, "deep-forced: " + _first_diff(edump, odump)
        assert etext == otext, "deep-forced: " + _first_diff(etext, otext)
        assert (ewarn[0], ewarn[1], ewarn[3]) == owarn


def test_fastmath_selftest_bound_covers_every_hot_numerator():
    """The self-test's numerator loop reaches 2 FASTDIV_MAX + 2 for every divisor: the hot path forms up to 2 (l_qseq - 1)."""
    K = kernel_constants()
    src = open(os.path.join(CSRC, "brc_kernels.cu")).read()
    body = src[src.index("fastmath_selftest_kernel("):]
    m = re.search(r"for\s*\(\s*int\s+a\s*=\s*threadIdx\.x\s*;\s*a\s*<=\s*([^;]+);", body)
    assert m, "numerator loop of fastmath_selftest_kernel not found"
    # the loop's bound for the smallest divisor must reach every numerator the hot path forms
    assert eval(m.group(1), {}, dict(K, b=1)) >= 2 * K["FASTDIV_MAX"] + 2


@pytest.mark.gpu
def test_fastmath_selftest_covers_every_hot_numerator():
    """brc_selftest_fastmath checks div_small against __fdiv_rn for every divisor b <= FASTDIV_MAX and every numerator up to
    2 FASTDIV_MAX + 2; a wrong quotient anywhere fails it."""
    from bam_readcount_b200.engine import Engine
    e = Engine()
    try:
        assert e.lib.brc_selftest_fastmath(e.h, kernel_constants()["FASTDIV_MAX"]) == 0
    finally:
        e.close()


@functools.lru_cache(maxsize=None)
def pool_case():
    """About 3000 sites at depth 60 whose reads carry random bases: every site holds four or five base classes, so the secondary
    pool needs several times the initial capacity brc_compute gives it."""
    c = cases.synthetic_case(L=3500, depth=60, seed=61, regions=((0, 201, 3200),), site_list=True, n_libs=8)
    b = c["batch"]
    rng = np.random.default_rng(61)
    codes = np.array([1, 2, 4, 8, 15], np.uint8)
    nib_hi, nib_lo = rng.choice(codes, b.seq.shape[0]), rng.choice(codes, b.seq.shape[0])
    b.seq = ((nib_hi << 4) | nib_lo).astype(np.uint8)
    return dict(c, name="pool")


def _initial_pool_cap(case, flags, n_slots):
    b = case["batch"]
    n_indel = int(np.isin(b.cigar & 0xF, (1, 2)).sum())
    rows = len(case["lib_names"]) if flags.get("per_lib") else 1
    return rows * n_slots // 8 + 2 * n_indel + 1024


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [dict(), dict(per_lib=True)], ids=["alllib", "perlib"])
def test_secondary_pool_grows_and_stays_exact(flags):
    from bam_readcount_b200.engine import Engine
    from test_site_filter import THRESHOLDS, select_lines
    case = pool_case()
    otext, odump, _ = cases.run_oracle(case, flags, site_list=True)
    # pipelined path (one borrowed push): its overflow falls through to the plain path, which grows the pool
    e = Engine(lib_names=case["lib_names"], **flags)
    try:
        name, clen, seq, wb = case["contigs"][0]
        e.set_reference(0, name, clen, seq, wb)
        tid, beg, end, sub = cases.region_reads(case, *case["regions"][0])
        e.begin_region(tid, beg, end, True)
        e.push_reads(sub)
        e.end_region()
        e.compute()
        pk = e.packed()
        assert pk.n_sec > _initial_pool_cap(case, flags, pk.n_slots), "the pool never outgrew its initial capacity: no retry ran"
        assert e.format_text(-1) == otext
    finally:
        e.close()
    etext, edump, _, _ = cases.run_engine(case, flags, site_list=True)
    assert edump == odump and etext == otext
    t2, _ = _engine_two_pushes(case, flags, True)              # copy path
    assert t2 == otext, _first_diff(t2, otext)
    from test_site_filter import _run
    for mc, mf in THRESHOLDS:                                  # filtered path
        text, _, _ = _run(case, flags, True, (mc, mf))
        assert text == select_lines(otext, mc, mf), (mc, mf)


@functools.lru_cache(maxsize=None)
def selection_cases():
    big = cases.synthetic_case(L=302000, depth=3, seed=71, n_libs=4,
                               regions=((0, 1, 300000), (0, 300001, 300100), (0, 300050, 300200), (0, 300201, 300300)), site_list=False)
    big = dict(big, name="sel_big")
    many = cases.synthetic_case(L=14000, depth=40, seed=72, n_libs=40, regions=tuple((0, 1000 + 40 * k, 1039 + 40 * k) for k in range(300)),
                                site_list=False)
    b = many["batch"]
    rng = np.random.default_rng(72)
    b.lib = b.lib.copy()
    b.lib[rng.random(b.n_reads) < 0.01] = 0xFFFF                # library-less reads
    return big, dict(many, name="sel_40libs")


@pytest.mark.gpu
@pytest.mark.parametrize("which", [0, 1], ids=["300k_sites", "40_libraries"])
def test_site_selection_at_scale(which):
    """More than 1024 scan partials (> 262 144 sites) with adjacent and overlapping argv regions; and -p with 40 libraries and
    library-less reads over 300 adjacent argv regions (the LIBRARY_UNAVAILABLE count of the selection's site pass).  That the
    deletion queue survives rows >= SEL_LAST_ROWS is test_site_selection_ships_the_queue_of_high_library_rows's."""
    from test_site_filter import THRESHOLDS, _run, select_lines
    K = kernel_constants()
    case = selection_cases()[which]
    flags = dict(per_lib=True) if which == 1 else dict()
    if which == 0:
        assert case["regions"][0][2] - case["regions"][0][1] + 1 > 1024 * K["SCAN_CTA"]
    else:
        assert len(case["lib_names"]) > K["SEL_LAST_ROWS"]
    otext, _, owarn = cases.run_oracle(case, flags, site_list=False)
    for mc, mf in THRESHOLDS:
        from bam_readcount_b200.engine import Engine
        e = Engine(lib_names=case["lib_names"], **flags)
        try:
            name, clen, seq, wb = case["contigs"][0]
            e.set_reference(0, name, clen, seq, wb)
            e.set_site_filter(mc, mf)
            for (ci, b1, e1) in case["regions"]:
                tid, beg, end, sub = cases.region_reads(case, ci, b1, e1)
                e.begin_region(tid, beg, end, False)
                e.push_reads(sub)
                e.end_region()
            e.compute()
            text = e.format_text(-1)
            w = e.warnings()
        finally:
            e.close()
        want = select_lines(otext, mc, mf)
        assert text == want, (mc, mf, _first_diff(text, want))
        if which == 1:
            assert owarn[2] > 0 and w[3] == owarn[2], (w, owarn)


@pytest.mark.gpu
def test_site_selection_ships_the_queue_of_high_library_rows():
    """boundary_cases.queue_rows: deletions of library rows >= SEL_LAST_ROWS anchored at an argv region's last site, a site no lower
    row covers and whose line fails the filter.  They print only in the next region, from the never-cleared deletion queue, so the
    selection must ship that site for those rows (sel_site_kernel's global reg_last branch); rows < 32 go through shared memory."""
    from test_site_filter import THRESHOLDS, _run, select_lines
    case = boundary_cases.queue_rows()
    flags = dict(per_lib=True)
    otext, odump, owarn = cases.run_oracle(case, flags, site_list=False)
    etext, _, ewarn, _ = cases.run_engine(case, flags, site_list=False, want_dump=False)
    assert etext == otext, _first_diff(etext, otext)
    assert (ewarn[0], ewarn[1], ewarn[3]) == owarn
    for a in case["probe"]["anchors"]:                          # the carried deletions do print in the next region
        assert any(ln.startswith(f"c\t{a + 2}\t") and "\t-" in ln for ln in otext.splitlines()), a
    for mc, mf in THRESHOLDS:
        text, _, _ = _run(case, flags, False, (mc, mf))
        want = select_lines(otext, mc, mf)
        assert text == want, (mc, mf, _first_diff(text, want))


def _device_batch(b, device):
    """The batch's arrays copied to the device (16 spare bytes behind the base and quality pools): a CReadBatch of device pointers
    and the tensors that own them."""
    import torch
    from bam_readcount_b200.engine import CReadBatch
    view = {np.dtype(np.uint16): np.int16, np.dtype(np.uint32): np.int32, np.dtype(np.uint64): np.int64}
    keep = []

    def dev(a, pad=0):
        a = np.ascontiguousarray(a)
        a = a.view(view.get(a.dtype, a.dtype))
        if pad:
            a = np.concatenate([a, np.zeros(pad, a.dtype)])
        t = torch.from_numpy(a).to(device)
        keep.append(t)
        return t.data_ptr()
    ptrs = [dev(b.tid), dev(b.pos), dev(b.flag), dev(b.mapq), dev(b.lib), dev(b.l_qseq), dev(b.nm), dev(b.sm), dev(b.cigar_off),
            dev(b.cigar), dev(b.seq_off), dev(b.seq, 64), dev(b.qual_off), dev(b.qual, 64)]
    return CReadBatch(b.n_reads, *ptrs), keep


@pytest.mark.gpu
def test_device_path_reports_pool_overflow_and_is_exact_when_replanned():
    """brc_plan_device with a secondary pool of 1024 records on the random-base pool case: brc_fetch_device_results must return
    BRC_E_OVERFLOW (the device path has no retry).  Re-planned with room, every raw accumulator equals the oracle's."""
    import torch
    from bam_readcount_b200.engine import BrcError, CRegion, Engine, admitted
    case = pool_case()
    _, odump, _ = cases.run_oracle(case, dict(), site_list=True)
    ci, b1, e1 = case["regions"][0]
    tid, beg, end, sub = cases.region_reads(case, ci, b1, e1)
    assert len(admitted(sub, tid, 10_000_000)) == sub.n_reads        # the device path admits every read it is given
    first_pos = max(beg - 1, 0)
    n_slots = int(min(end, int(sub.ref_end().max()))) - first_pos
    dev = torch.device("cuda", 0)
    cb, keep = _device_batch(sub, dev)
    name, clen, seq, wb = case["contigs"][0]
    e = Engine(lib_names=case["lib_names"])
    try:
        e.set_reference(tid, name, clen, seq, wb)
        s = torch.cuda.Stream(device=dev)
        for cap in (1024, 1 << 20):
            e.plan_device([CRegion(tid, beg, end, 1, 0, sub.n_reads, 0, first_pos, n_slots)], sub.n_reads, cap)
            e.run_device(cb, None, s.cuda_stream)
            if cap == 1024:
                with pytest.raises(BrcError) as err:
                    e.fetch_device_results(s.cuda_stream)
                assert err.value.status == -8          # BRC_E_OVERFLOW
            else:
                res = e.fetch_device_results(s.cuda_stream)
                edump = res.dump(sub, {tid: (wb, seq)})
                assert edump == odump, _first_diff(edump, odump)
    finally:
        e.close()
    del keep


@pytest.mark.gpu
def test_bgzf_record_scan_over_more_than_one_scan_level():
    """A synth_cb sample of 1500 blocks decoded on the device as ONE span: its record framing runs the shared exclusive scan over
    more than 1024 partials (> 262 144 records).  Every array equals bamio's host decode."""
    import tempfile
    from bam_readcount_b200 import bamio, synth_cb
    from bam_readcount_b200.engine import Engine
    from oracle.oracle import REF_SAMTOOLS
    if not os.path.exists(REF_SAMTOOLS):
        pytest.skip("oracle/_ref/samtools not built")
    tmp = tempfile.mkdtemp()
    sp = synth_cb.Spec(seed=31, contig_len=1280 * 1600)
    info = synth_cb.write_sample_bam(sp, 0, 0, 1500, tmp, REF_SAMTOOLS)
    hdr, host = bamio.read_bam(info["bam"])
    rg_lib = {rg: hdr.lib_of_rg(rg) for rg in hdr.rg_lb}
    span = bamio.bam_span(info["bam"], bamio.BaiIndex(info["bam"] + ".bai"), 0, 0, info["length"], rg_lib)
    e = Engine(per_lib=True, lib_names=hdr.lib_names)
    try:
        got = e.decode_bam_span(span)
    finally:
        e.close()
    K = kernel_constants()
    assert got.n_reads > 1024 * K["SCAN_CTA"]
    want = host.select(host.fetch(0, 0, info["length"]))
    assert got.n_reads == want.n_reads == host.n_reads
    for k in ("pos", "flag", "mapq", "lib", "l_qseq", "nm", "sm", "cigar_off", "cigar", "seq_off", "seq", "qual_off", "qual"):
        g, w = np.asarray(getattr(got, k)), np.asarray(getattr(want, k))
        assert g.shape == w.shape and np.array_equal(g, w.astype(g.dtype)), k
