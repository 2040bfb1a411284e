"""K0 (read_precompute_kernel, brc_kernels.cu) against its model, field by field: every ReadDesc and every tile range.

The model is kernel_model.k0_descriptors: fetch_func's five values and bam_endpos from the oracle's C ports, the other fields
restated from brc_device.cuh.  A failure names the first read that differs, the field, both values and the read's shape.

CPU
  audit   tests/k0_cases.py reaches the edges of K0's code: every (read, reference) nibble phase pair on the staged and the
          global path, a mismatch at every lane of a 16-base step, runs of mismatches across a step and across M D / N M
          (one run) and M I M (two), the `keep` mask binding for 1-15 bases left, every (read code, reference code) pair, each
          quality lead on both strands and both paths with the Q2 scan's first and last masks binding, every byte value
          stopping the scan, the reference staged and not within one read, the walk reaching chrom_len in both region modes.
          Audited twice: on the case's own pools (the borrowed push and brc_run_device read them) and on the pools
          brc_push_read builds when it copies the reads.
GPU
  the device's descriptors and tile ranges equal the model's on the K0 case, every boundary case, the contigs near 2^31, a
  synthetic case under -q 20 -b 20 -p, the edge fuzz cases, test.bam and a C4 window of the generator; the K0 case through
  every launch path: the pipelined push at several chunk counts, two pushes (copied pools), several regions on two contigs,
  and brc_run_device with the base or quality pool starting 1-3 bytes into its allocation.  Each push asserts from the
  launch count that the engine took the path (pipelined or plain) the model assumes."""
from __future__ import annotations

import dataclasses
import functools
import os

import numpy as np
import pytest

import boundary_cases
import cases
import edge32_cases
import edge_cases
import k0_cases
from kernel_model import DESC, FM_DEAD, k0_blocks, k0_descriptors, kernel_constants
from pipeline_cases import pipe_launches, pipe_plan

QBP = dict(min_mapq=20, min_bq=20, per_lib=True)
FLAG_SETS = {"default": dict(), "q20b20p": QBP}


# ---------------------------------------------------------------------------------------------------------------------------
# CPU: the K0 case reaches K0's edges
# ---------------------------------------------------------------------------------------------------------------------------
def _q2_scan(qual, qoff, lq, reverse, first_mask=True, last_mask=True):
    """K0's Q2 scan over the aligned words holding the read's qualities (bytes outside the pool read as 0)."""
    lead = qoff & 3
    wl = (lq - 1 + lead) >> 2
    fm, lm = (~0 << (8 * lead)) & 0xFFFFFFFF, 0xFFFFFFFF >> (8 * (3 - ((lq - 1 + lead) & 3)))
    ws = range(0, wl + 1) if reverse else range(wl, -1, -1)
    for w in ws:
        ne = 0
        for b in range(4):
            k = qoff - lead + 4 * w + b
            v = int(qual[k]) if k < qual.shape[0] else 0
            ne |= (v != 2) << (8 * b + 7)
        if w == 0 and first_mask:
            ne &= fm
        if w == wl and last_mask:
            ne &= lm
        if ne:
            byte = ((ne & -ne).bit_length() - 1 if reverse else ne.bit_length() - 1) >> 3
            return 4 * w + byte - lead - 1
    return -1


def copied_pools(b):
    """The batch with its pools laid out as brc_push_read copies them: per read (l_qseq + 1) / 2 base bytes and l_qseq
    qualities, back to back."""
    from bam_readcount_b200.batch import ReadBatch
    so, qo = b.seq_off.astype(np.int64), b.qual_off.astype(np.int64)
    lq = b.l_qseq.astype(np.int64)
    seq = np.concatenate([b.seq[so[i]:so[i] + (lq[i] + 1) // 2] for i in range(b.n_reads)])
    qual = np.concatenate([b.qual[qo[i]:qo[i] + lq[i]] for i in range(b.n_reads)])
    cum = lambda x: np.concatenate([[0], np.cumsum(x)]).astype(np.uint64)   # noqa: E731
    return dataclasses.replace(b, seq=seq, seq_off=cum((lq + 1) // 2), qual=qual, qual_off=cum(lq))


LAYOUTS = ("own", "copied")


@functools.lru_cache(maxsize=None)
def k0_reach(layout):
    """What the K0 case makes K0 do, per target (sets of what was reached), on the pools K0 reads: the case's own ("own": the
    borrowed push, which runs compute_pipelined, and brc_run_device) or those brc_push_read builds ("copied": the reads of a
    push that is not borrowed)."""
    case = k0_cases.k0_case()
    contig = case["contigs"][0]
    _, chrom_len, seq, wb = contig
    refc = np.concatenate([k0_cases.NT16[np.frombuffer(seq, np.uint8)], np.full(64, 15, np.uint8)])
    R = {k: set() for k in ("phase_staged", "phase_global", "lane", "step_run", "op_run", "ins_split", "keep", "codes",
                            "lead", "first_mask", "last_mask", "stop_byte", "lq", "q2_run", "tpi", "ref_staged_mix",
                            "hit_nul", "ref_unstaged_span", "n_cigar_wide", "fastdiv")}
    for sl in case["modes"]:
        _, _, _, b, _, _, _ = cases.region_geometry(case, case["regions"][0])
        if layout == "copied":
            b = copied_pools(b)
        nib = np.empty(2 * b.seq.shape[0], np.uint8); nib[0::2] = b.seq >> 4; nib[1::2] = b.seq & 15
        so, qo, co = (x.astype(np.int64) for x in (b.seq_off, b.qual_off, b.cigar_off))
        d, _, _ = k0_descriptors(b, [dict(ref=0, site_list=sl, first_pos=0, n_slots=0, read_lo=0, read_hi=b.n_reads)], [contig], {})
        for blk in k0_blocks(b, case, site_list=sl, ops=True):
            path = "staged" if blk["staged"] else "global"
            for i, ops in zip(range(blk["r0"], blk["r1"]), blk["ops"]):
                rev = bool(b.flag[i] & 16)
                lq = int(b.l_qseq[i])
                mms = []                                      # (read offset, op index)
                staged_ops = {o["ref_staged"] for o in ops if o["j"] < o["jend"]}
                if staged_ops == {True, False}:
                    R["ref_staged_mix"].add(path)
                if blk["staged"] and not blk["ref_staged"] and blk["span"] > 2 * kernel_constants()["K0_REF_CAP"]:
                    R["ref_unstaged_span"].add(True)
                for k, o in enumerate(ops):
                    if o["hit_nul"]:
                        R["hit_nul"].add((sl, "straddle" if o["wrel"] + wb < chrom_len else "at_or_past"))
                    if sl and o["wrel"] + wb > chrom_len:
                        R["hit_nul"].add((sl, "skipped_past"))
                    j, jend = o["j"], o["jend"]
                    if j >= jend:
                        continue
                    t0 = 2 * so[i] + o["rp"]
                    if blk["staged"] and o["ref_staged"]:
                        R["phase_staged"].add(((t0 + j) % 8, (o["wrel"] + j) % 8))
                    elif not blk["staged"]:
                        R["phase_global"].add(((t0 + j) % 8, (o["wrel"] + j) % 8))
                    jj = np.arange(j, jend)
                    r = nib[t0 + jj]; f = refc[o["wrel"] + jj]
                    R["codes"].update(zip(r.tolist(), f.tolist()))
                    mm = (r != f) & (f != 15) & (r != 0)
                    for x in jj[mm].tolist():
                        R["lane"].add((path, (x - j) % 16))
                        mms.append((o["rp"] + x, k, x == j, x == jend - 1))
                        if mm[x - j - 1] and x > j and (x - j) % 16 == 0:
                            R["step_run"].add(path)
                    nv = (jend - j) % 16
                    if nv:
                        last = j + (jend - j) // 16 * 16
                        for lane in range(nv, 16):
                            x = last + lane
                            tr = t0 + x
                            rr = int(nib[tr]) if tr < nib.shape[0] else 0
                            ff = int(refc[o["wrel"] + x]) if o["wrel"] + x < refc.shape[0] else 15
                            if rr != ff and ff != 15 and rr != 0:
                                R["keep"].add((path, nv))
                                break
                for (p1, k1, _, end1), (p2, k2, start2, _) in zip(mms, mms[1:]):
                    if k2 == k1 + 1 and end1 and start2:
                        R["op_run" if p2 == p1 + 1 else "ins_split"].add(path)
                # qualities
                lead = int(qo[i]) & 3
                R["lead"].add((path, lead, rev))
                if lq > 0:
                    q2 = _q2_scan(b.qual, int(qo[i]), lq, rev)
                    assert q2 == d["q2"][i], (i, q2, d["q2"][i])      # the word scan restates fetch_func's byte loop
                    if _q2_scan(b.qual, int(qo[i]), lq, rev, first_mask=False) != q2:
                        R["first_mask"].add((path, rev))
                    if _q2_scan(b.qual, int(qo[i]), lq, rev, last_mask=False) != q2:
                        R["last_mask"].add((path, rev))
                    stop = (q2 + 1) if q2 >= 0 or (rev and lq and b.qual[qo[i]] != 2) else None
                    if stop is not None and 0 <= stop < lq:
                        R["stop_byte"].add(int(b.qual[qo[i] + stop]))
                    run = (q2 + 1 if q2 >= 0 else 0) if rev else (lq - 1 - (q2 + 1) if q2 >= 0 else 0)
                    ql = b.qual[qo[i]:qo[i] + lq]
                    if (ql == 2).all():
                        run = lq
                    R["q2_run"].add((lq, run))
                R["lq"].add(lq)
                t = int(d["tpi"][i]); q2 = int(d["q2"][i]); lc = int(d["lclip"][i])
                if rev:
                    R["tpi"].add("rev_left_clip" if t == lc > 0 and q2 < lc else "rev_q2" if t == q2 > lc else "rev_none")
                else:
                    R["tpi"].add("fwd_right_clip" if t < lq - 1 and (q2 == -1 or q2 > t) else "fwd_q2" if t == q2 < lq - 1 else "fwd_none")
                nc = int(co[i + 1] - co[i])
                if nc > 0xFFFF:
                    R["n_cigar_wide"].add(True)
                R["fastdiv"].update(x for x in (("lq", lq), ("clen", int(d["clen"][i]))) if x[1] in (2048, 2049))
    return R


def _missed(name, want, got):
    miss = sorted(set(want) - set(got), key=repr)
    assert not miss, f"{name}: missed {miss[:12]}{' ...' if len(miss) > 12 else ''} ({len(miss)} of {len(set(want))})"


@pytest.mark.parametrize("layout", LAYOUTS)
def test_k0_case_reaches_every_target(layout):
    R = k0_reach(layout)
    pairs = [(a, b) for a in range(8) for b in range(8)]
    _missed("phase pairs, staged bases and reference", pairs, R["phase_staged"])
    _missed("phase pairs, bases and reference from global memory", pairs, R["phase_global"])
    _missed("mismatch lanes", [(p, k) for p in ("staged", "global") for k in range(16)], R["lane"])
    _missed("runs across a step", ["staged", "global"], R["step_run"])
    _missed("runs across M D M / M N M", ["staged", "global"], R["op_run"])
    _missed("runs split by M I M", ["staged", "global"], R["ins_split"])
    _missed("keep mask binding at n bases left", [("staged", n) for n in range(1, 16)], R["keep"])
    _missed("(read code, reference code) pairs", [(a, b) for a in range(16) for b in range(16)], R["codes"])
    _missed("quality lead x strand", [(p, l, r) for p in ("staged", "global") for l in range(4) for r in (False, True)], R["lead"])
    _missed("Q2 first-word mask binding", [(p, r) for p in ("staged", "global") for r in (False, True)], R["first_mask"])
    _missed("Q2 last-word mask binding", [(p, r) for p in ("staged", "global") for r in (False, True)], R["last_mask"])
    _missed("byte values stopping the Q2 scan (every byte but 2)", [v for v in range(256) if v != 2], R["stop_byte"])
    _missed("l_qseq", list(range(1, 13)) + [150, 151, 2048, 2049], R["lq"])
    _missed("Q2 runs of no base and of the whole read", [(l, 0) for l in range(1, 13)] + [(l, l) for l in range(1, 13)], R["q2_run"])
    _missed("three_prime_index clamps", ["rev_left_clip", "rev_q2", "fwd_right_clip", "fwd_q2"], R["tpi"])
    _missed("reference staged and not within one read", ["staged"], R["ref_staged_mix"])
    _missed("block spanning more than 2 K0_REF_CAP bases", [True], R["ref_unstaged_span"])
    _missed("the walk reaching chrom_len", [(m, w) for m in (False, True) for w in ("straddle", "at_or_past")] + [(True, "skipped_past")],
            R["hit_nul"])
    _missed("more than 65,535 CIGAR ops", [True], R["n_cigar_wide"])
    _missed("FASTDIV_MAX and one past it", [("lq", 2048), ("lq", 2049), ("clen", 2048), ("clen", 2049)], R["fastdiv"])


def test_model_tile_ranges_equal_the_per_read_loop():
    """The vectorised tile ranges against the obvious per-read loop over every tile a read overlaps."""
    from kernel_model import tile_ranges
    T = kernel_constants()["TILE"]
    case = k0_cases.k0_case()
    _, _, _, b, fp, ns, _ = cases.region_geometry(case, case["regions"][0])
    e = b.ref_end()
    want = {}
    for i in range(b.n_reads):
        a, z = max(int(b.pos[i]), fp), min(int(e[i]), fp + ns)
        for t in range((a - fp) // T, (z - 1 - fp) // T + 1) if z > a and not b.flag[i] & 4 else ():
            lo, hi = want.get(t, (2 ** 31 - 1, 0))
            want[t] = (min(lo, i), max(hi, i + 1))
    got = tile_ranges(b, fp, fp + ns)
    assert got == [want.get(t, (0, 0)) for t in range(len(got))]


# ---------------------------------------------------------------------------------------------------------------------------
# GPU: the device against the model
# ---------------------------------------------------------------------------------------------------------------------------
FIELDS = DESC.names
FLOATS = ("nmfrac", "fl", "rcp_l", "rcp_clen", "fclen")


def _describe(b, i, offsets, launches, contig, site_list):
    co = b.cigar_off.astype(np.int64)
    ops = "".join(f"{int(c) >> 4}{'MIDNSHP=XB'[int(c) & 15] if int(c) & 15 < 10 else '?'}" for c in b.cigar[co[i]:co[i + 1]][:40])
    blk = [x for x in k0_blocks(b, dict(contigs=[contig], site_list=site_list), launches) if x["r0"] <= i < x["r1"]] if contig else []
    stage = (f"block [{blk[0]['r0']}, {blk[0]['r1']}) staged={blk[0]['staged']} ref_staged={blk[0]['ref_staged']}" if blk
             else "block staging not modelled")
    q = int(np.asarray(offsets.get("qual", b.qual_off))[i])
    return (f"pos {int(b.pos[i])} cigar {ops}{'...' if co[i + 1] - co[i] > 40 else ''} flag {int(b.flag[i])} "
            f"{'reverse' if b.flag[i] & 16 else 'forward'} l_qseq {int(b.l_qseq[i])} qual_off%4 {q % 4} {stage}")


def assert_desc_equal(got, want_desc, want_lo, want_hi, b, what, offsets=None, launches=None, contig=None, site_list=False):
    desc, lo, hi = got
    assert desc.shape[0] == want_desc.shape[0], f"{what}: {desc.shape[0]} descriptors, the model has {want_desc.shape[0]}"
    g = np.ascontiguousarray(desc).view(DESC).reshape(-1)
    for f in FIELDS:
        x, y = g[f], want_desc[f]
        if f in FLOATS:
            bad = (x.view(np.uint32) != y.view(np.uint32)) & ~(np.isnan(x) & np.isnan(y))
        else:
            bad = x != y
        if bad.any():
            i = int(np.nonzero(bad)[0][0])
            raise AssertionError(f"{what}: read {i}, field {f}: kernel {x[i]!r}, model {y[i]!r} ({int(bad.sum())} reads differ); "
                                 + _describe(b, i, offsets or {}, launches, contig, site_list))
    for name, x, y in (("tile_lo", lo, want_lo), ("tile_hi", hi, want_hi)):
        assert x.shape == y.shape, f"{what}: {x.shape[0]} tiles, the model has {y.shape[0]}"
        bad = np.nonzero(x != y)[0]
        assert not bad.size, f"{what}: {name}[{int(bad[0])}]: kernel {int(x[bad[0]])}, model {int(y[bad[0]])} ({bad.size} tiles differ)"


def _borrowable(part, cnt):
    """brc_push_reads keeps a view of the first batch pushed after a reset when every read is admitted as is (scan_batch)."""
    e = part.ref_end()
    dup_zero = bool(np.any((e[1:] <= part.pos[1:]) & (np.diff(part.pos) == 0)))
    return (0 < part.n_reads < cnt and not (part.flag & 4).any() and bool(np.all(np.diff(part.pos) >= 0))
            and len(set(part.tid.tolist())) == 1 and not dup_zero)


def _pushed(case, site_list, regions, push, flags):
    """The reads the engine holds after push_regions, the model's regions and the pool offsets the engine used: a borrowed
    first push keeps its own pools (rebased to 0 once more reads follow), every read pushed after it is copied (brc_push_read:
    its CIGAR ops, (l_qseq + 1) / 2 base bytes and l_qseq qualities appended)."""
    from bam_readcount_b200.engine import admitted
    from bam_readcount_b200.batch import ReadBatch
    subs, regs, lo = [], [], 0
    cnt = flags.get("max_cnt", 10_000_000)
    for ci, b1, e1 in regions:
        tid, beg, end, sub = cases.region_reads(case, ci, b1, e1)
        keep = admitted(sub, tid, cnt)
        s = sub.select(keep)
        first_pos = max(beg - 1, 0)
        max_end = max([first_pos] + s.ref_end().tolist())
        regs.append(dict(ref=ci, site_list=site_list, first_pos=first_pos, n_slots=max(0, min(end, max_end) - first_pos),
                         read_lo=lo, read_hi=lo + s.n_reads))
        subs.append((sub, s))
        lo += s.n_reads
    b = ReadBatch.concat([s for _, s in subs])
    sub0 = subs[0][0]
    first = sub0 if push == "one" else sub0.select(np.arange(sub0.n_reads // 2))
    n_b = first.n_reads if _borrowable(first, cnt) else 0
    if n_b == b.n_reads:
        return b, regs, case["contigs"], {}, len(regions) == 1
    offsets = {}
    for name, size in (("cigar", np.diff(b.cigar_off.astype(np.int64))), ("seq", (b.l_qseq.astype(np.int64) + 1) // 2),
                       ("qual", b.l_qseq.astype(np.int64))):
        own = getattr(b, name + "_off").astype(np.int64)
        off = np.concatenate([own[:n_b + 1] - own[0], own[n_b] - own[0] + np.cumsum(size[n_b:])])
        offsets[name] = off.astype(np.uint64)
    return b, regs, case["contigs"], offsets, False


def pipe_chunks(b):
    """The chunk count compute_pipelined picks for a borrowed batch (issue_h2d_chunks): ~64 MiB of input per chunk, at most
    32, at least 4096 reads each; BRC_PIPE_CHUNKS overrides it."""
    n = b.n_reads
    in_bytes = n * 21 + 3 * (n + 1) * 8 + int(b.cigar_off[n]) * 4 + int(b.seq_off[n]) + int(b.qual_off[n])
    k = min(min(32, max(1, in_bytes >> 26)), max(1, n // 4096))
    if os.environ.get("BRC_PIPE_CHUNKS"):
        k = max(1, min(int(os.environ["BRC_PIPE_CHUNKS"]), max(1, n)))
    return k


def k0_path(b, regs, pipelined):
    """(launch count, K0 launches) of the run the model assumes: compute_pipelined cuts a borrowed single-region batch into
    chunks and launches K0 once per chunk (pipeline_cases.pipe_plan); every other push runs K0 once over all reads.  The deep-site
    kernel is off (no_deep_kernel)."""
    T = kernel_constants()["TILE"]
    n_tiles = sum((g["n_slots"] + T - 1) // T for g in regs)
    if pipelined:
        plan = pipe_plan(b.pos, regs[0]["first_pos"], n_tiles, pipe_chunks(b))
        return pipe_launches(plan), [(a, z) for a, z, _, _ in plan]
    return 2 + (n_tiles > 0), [(0, b.n_reads)]


def h2d_bytes(b, offsets, path):
    """Bytes brc_compute copies to the device (brc_last_h2d_bytes) on `path`.  "pipelined" leaves out the columns the admission
    scan found regular (offsets of a fixed stride, one l_qseq, one SM value: rebuilt on the device); "plain" copies every
    column of the engine's pools and the region of each read; "overflow" is the plain path run on a borrowed batch, after the
    secondary pool of the pipelined run overflowed (brc_compute falls through to it: every column, no regions)."""
    n = b.n_reads
    off = {k: np.asarray(offsets.get(k, getattr(b, k + "_off")), np.int64) for k in ("cigar", "seq", "qual")}
    pools = 4 * int(off["cigar"][n] - off["cigar"][0]) + int(off["seq"][n] - off["seq"][0]) + int(off["qual"][n] - off["qual"][0])
    if path != "pipelined":
        return 21 * n + 3 * 8 * (n + 1) + pools + (4 * n if path == "plain" else 0)
    regular = lambda o: bool(np.all(o[1:] - o[0] == np.arange(1, n + 1) * (o[1] - o[0])))   # noqa: E731
    skip = n >= 2 and not os.environ.get("BRC_NO_H2D_ELISION")
    return (21 * n + 8 * (n + 1) + pools - (skip and len(set(b.l_qseq.tolist())) == 1) * 4 * n
            - (skip and len(set(b.sm.tolist())) == 1) * 4 * n + 8 * (n + 1) * (2 - skip * (regular(off["seq"]) + regular(off["qual"]))))


def run_push(case, flags, site_list, *, regions=None, push="one"):
    """One compute of the case's reads pushed by push_regions: (the device's descriptors, the model's, the reads as the engine
    holds them, the pool offsets it used, the K0 launches).  Asserts from the launch count and the bytes copied that the engine
    took the path the model assumes: pipelined for a borrowed single-region batch, unless its secondary pool overflowed there and
    the plain path computed it again (which then launched K0 last), plain for every other push."""
    regions = case["regions"] if regions is None else regions
    with cases.open_engine(case, flags) as e:
        cases.push_regions(e, case, site_list, regions, push=push)
        e.compute()
        got = e.read_descriptors()
        launched, copied = e.launch_count(), e.h2d_bytes()
    b, regs, refs, offsets, pipelined = _pushed(case, site_list, regions, push, flags)
    path = "pipelined" if pipelined else "plain"
    if pipelined and copied != h2d_bytes(b, offsets, path) and copied == h2d_bytes(b, offsets, "overflow"):
        pipelined, path = False, "overflow"     # the pool outgrew its first capacity: the plain path ran K0 last
    n_launch, launches = k0_path(b, regs, pipelined)
    assert launched == n_launch, f"{launched} kernel launches, {n_launch} expected: the engine did not take the {path} path"
    assert copied == h2d_bytes(b, offsets, path), f"{copied} bytes copied, {h2d_bytes(b, offsets, path)} expected on the {path} path"
    want = k0_descriptors(b, regs, refs, flags, offsets)
    return got, want, b, offsets, launches


def check_push(case, flags, site_list, what, *, regions=None, push="one"):
    """run_push, its descriptors compared with the model's; returns the K0 launches."""
    got, want, b, offsets, launches = run_push(case, flags, site_list, regions=regions, push=push)
    single = len(case["regions"] if regions is None else regions) == 1
    assert_desc_equal(got, *want, b, what, offsets, launches, case["contigs"][0] if single else None, site_list)
    return launches


@pytest.fixture(autouse=True)
def no_deep_kernel(monkeypatch):
    """The deep-site kernel reads the descriptors and writes none; off, a run's launch count tells its path."""
    monkeypatch.setenv("BRC_DEEP_MIN_READS", str(0x7FFFFFFF))


def _first_modes(case):
    return case.get("modes", (case["site_list"],))


@functools.lru_cache(maxsize=None)
def fixture_cases():
    """{name: (case, flags, site_list)} of the families checked pushed in one piece: the pipelined path where brc_push_reads
    borrows the batch (the K0 case among them), the plain one where it copies it (a case holding reads a push does not
    admit, or several regions)."""
    out = {}
    k0 = k0_cases.k0_case()
    for sl in k0["modes"]:
        for fname, fl in FLAG_SETS.items():
            out[f"k0_{'sitelist' if sl else 'argv'}_{fname}"] = (k0, fl, sl)
    for c in boundary_cases.all_cases():
        for fname in ("default", "perlib_ic_q20b20"):
            out[f"{c['name']}_{fname}"] = (c, boundary_cases.FLAG_SETS[fname], _first_modes(c)[0])
    for k in (0, 3):
        c = edge32_cases.contig_end_2_31(k)
        out[c["name"]] = (c, {}, _first_modes(c)[0])
        s = edge32_cases.site_lines(c)
        out[s["name"]] = (s, {}, s["site_list"])
    syn = cases.synthetic_case(L=40000, depth=30, seed=31, regions=((0, 2000, 38000),), n_libs=4)
    out["synthetic_q20_b20_p"] = (syn, QBP, syn["site_list"])
    for c in edge_cases.all_cases():
        for fname in ("default", "q20b20"):
            fl = c["flag_sets"][fname]
            out[f"{c['name']}_{fname}"] = (c, fl, c["site_list"])
    tb = cases.testbam_case()
    out["test_bam"] = (tb, {}, True)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(fixture_cases()))
def test_k0_descriptors_equal_model(name):
    case, flags, sl = fixture_cases()[name]
    check_push(case, flags, sl, name)


@pytest.mark.gpu
@pytest.mark.parametrize("chunks", [3, 7])
def test_k0_pipelined_chunks(chunks, monkeypatch):
    """compute_pipelined at chunk counts whose K0 launches start at reads that are not multiples of K0_READS (their staged
    ranges then start mid-pool).  The K0 case is borrowed as pushed; run_push asserts the launch count of that path."""
    monkeypatch.setenv("BRC_PIPE_CHUNKS", str(chunks))
    case = k0_cases.k0_case()
    for sl in case["modes"]:
        for fname, fl in FLAG_SETS.items():
            launches = check_push(case, fl, sl, f"{chunks} chunks, {fname}, site_list={sl}")
            assert len(launches) == chunks, f"not the pipelined path: {launches}"
            assert any(a % kernel_constants()["K0_READS"] for a, _ in launches), launches


@pytest.mark.gpu
def test_k0_two_pushes_copied_pools():
    case = k0_cases.k0_case()
    for sl in case["modes"]:
        for fname, fl in FLAG_SETS.items():
            check_push(case, fl, sl, f"two pushes, {fname}, site_list={sl}", push="halves")


def two_contig_case():
    """The K0 case on two contigs, in several regions of each: one compute with region_of_read and no reference staging."""
    from bam_readcount_b200.batch import ReadBatch
    c = k0_cases.k0_case()
    b = c["batch"]
    b2 = dataclasses.replace(b, tid=np.ones_like(b.tid))
    name, L, seq, wb = c["contigs"][0]
    we = wb + len(seq)
    cuts = [wb + 2, wb + 3000, wb + 3001, wb + 12000, wb + 40000, we]
    regions = [(0, cuts[0], cuts[1]), (0, cuts[2], cuts[3]), (0, cuts[3] + 5, cuts[4]), (1, cuts[0] + 500, cuts[3]),
               (1, cuts[4], cuts[5])]
    return dict(name="k0_two_contigs", contigs=[c["contigs"][0], ("k0b", L, seq, wb)], batch=ReadBatch.concat([b, b2]),
                regions=regions, site_list=False, lib_names=c["lib_names"])


@pytest.mark.gpu
def test_k0_several_regions_on_two_contigs():
    case = two_contig_case()
    for sl in (False, True):
        for fname, fl in FLAG_SETS.items():
            check_push(case, fl, sl, f"several regions, {fname}, site_list={sl}")


@pytest.mark.gpu
@pytest.mark.parametrize("pool", ["qual", "seq"])
@pytest.mark.parametrize("lead", [1, 2, 3])
def test_k0_device_path_pool_leads(pool, lead):
    """brc_plan_device / brc_run_device with one pool starting `lead` bytes into its allocation (every read, the placed unmapped
    one included: the device path admits all it is given)."""
    import torch
    from bam_readcount_b200.engine import CRegion
    case = k0_cases.k0_case(unmapped=True)
    region = case["regions"][0]
    dev = torch.device("cuda", 0)
    for sl in case["modes"]:
        tid, beg, end, sub, first_pos, n_slots, _ = cases.region_geometry(case, region)
        cb, keep = cases.device_batch(sub, dev, lead=(pool, lead))
        with cases.open_engine(case, QBP) as e:
            s = torch.cuda.Stream(device=dev)
            e.plan_device([CRegion(tid, beg, end, int(sl), 0, sub.n_reads, 0, first_pos, n_slots)], sub.n_reads, 1 << 20)
            e.run_device(cb, None, s.cuda_stream)
            got = e.read_descriptors()
        del keep
        off = {pool: getattr(sub, pool + "_off").astype(np.uint64) + np.uint64(lead)}
        want = k0_descriptors(sub, [dict(ref=0, site_list=sl, first_pos=first_pos, n_slots=n_slots, read_lo=0, read_hi=sub.n_reads)],
                              case["contigs"], QBP, off)
        unmapped = (sub.flag & 4) != 0
        assert unmapped.any() and (want[0]["fm"][unmapped] & FM_DEAD).all()
        assert_desc_equal(got, *want, sub, f"device path, {pool} pool lead {lead}, site_list={sl}", off, None, case["contigs"][0], sl)


@pytest.mark.gpu
def test_k0_descriptors_c4_window():
    """A C4 window of the generator (bench.py's workload), its reads generated in HBM."""
    import torch
    from bam_readcount_b200 import stream as st
    from bam_readcount_b200 import synth_cb
    from bench import CONFIGS
    cfg = CONFIGS["c4"]
    spec = synth_cb.Spec(seed=1234, mode=synth_cb.WGS, n_libs=8, contig_len=cfg["contig_blocks"] * synth_cb.BLOCK_BP, n_contigs=1)
    windows = st.wgs_windows(spec, cfg["windows_per_contig"])
    w = windows[len(windows) // 2]
    r = st.WindowRunner(spec, spec.window_reads(w.blk_lo, w.blk_hi), torch.device("cuda", 0), cfg["flags"])
    try:
        r.launch(w)
        torch.cuda.synchronize()
        got = r.eng.read_descriptors()
        b = r.dw.to_host()
    finally:
        r.close()
    L = st.reference_length(spec)
    contig = (f"chr{w.contig + 1}", L, spec.ref_host(w.contig, 0, L), 0)
    reg = dict(ref=0, site_list=False, first_pos=w.first_pos, n_slots=w.n_slots, read_lo=0, read_hi=b.n_reads)
    want = k0_descriptors(b, [reg], [contig], cfg["flags"])
    assert_desc_equal(got, *want, b, "c4 window", {}, None, contig, False)
