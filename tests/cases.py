"""Shared parity-test cases: deterministic inputs + runners for the oracle and the CUDA engine.

A case is a dict: contigs [(name, length, ref_bytes, win_beg)], batch (all reads, file order),
regions [(contig_index, beg1, end1)] in 1-based inclusive coordinates as a user would write
them, ``site_list`` (True: -l loop, False: argv regions), flags, lib_names.

The harness every parity test goes through: ``run_oracle`` / ``run_oracle_cached``, ``run_engine`` (one brc_compute over the
case's regions) and ``run_engine_per_region`` (one per region, deletion queue carried), ``assert_same`` and ``first_diff`` to
compare them, ``device_batch`` / ``run_device`` for the device-resident path, ``assert_anchor`` for the reference binary's
SHA-256.

The fixtures of the tests that run executables: ``cli`` / ``samtools`` / ``check_program`` build or find them;
``write_fasta``, ``write_testbam_fasta``, ``write_bam``, ``sam_to_bam`` and ``synthetic_bam`` write their inputs;
``load_golden_text`` / ``golden_texts`` read the committed outputs.
"""
from __future__ import annotations

import atexit
import contextlib
import dataclasses
import functools
import gzip
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
from typing import NamedTuple, Optional

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bam_readcount_b200 import synth  # noqa: E402
from bam_readcount_b200.batch import BatchBuilder, ReadBatch, TAG_ABSENT  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
CRAM_DATA = os.path.join(ROOT, "oracle", "_ref", "test-data")      # the reference's test-data, CRAM fixture included
DECODE_ONLY = dict(os.environ, BRC_CLI_DECODE_ONLY="1")            # brc-readcount prints per-region record summaries, no device

FLAG_SETS = {
    "default": dict(),
    "q20b20": dict(min_mapq=20, min_bq=20),
    "ic": dict(insertion_centric=True),
    "perlib": dict(per_lib=True),
    "perlib_ic_q20b20": dict(per_lib=True, insertion_centric=True, min_mapq=20, min_bq=20),
    "d5": dict(max_cnt=5),
}


def flags_to_argv(fl: dict) -> list:
    a = []
    if "min_mapq" in fl:
        a += ["-q", str(fl["min_mapq"])]
    if "min_bq" in fl:
        a += ["-b", str(fl["min_bq"])]
    if "max_cnt" in fl:
        a += ["-d", str(fl["max_cnt"])]
    if fl.get("per_lib"):
        a += ["-p"]
    if fl.get("insertion_centric"):
        a += ["-i"]
    return a


def synthetic_case(L=30000, depth=30, seed=7, regions=((0, 3000, 23000),), site_list=False, n_libs=8):
    ref = synth.synth_reference(L, seed)
    batch = synth.synth_reads(ref, depth, seed=seed, n_libs=n_libs)
    return dict(name=f"syn_L{L}_d{depth}_s{seed}", contigs=[("chr1", L, ref.tobytes(), 0)], batch=batch,
                regions=list(regions), site_list=site_list, lib_names=[f"lib{i}" for i in range(n_libs)])


def deep_case(n_sites=3, depth=5000, seed=5, n_libs=8, L=2000):
    ref = synth.synth_reference(L, seed)
    sites = np.linspace(400, L - 400, n_sites).astype(np.int64)
    batch, bounds = synth.synth_deep_panel(ref, sites, depth, seed=seed, n_libs=n_libs)
    # one BAM: merge all groups and sort by position (stable) like a coordinate-sorted file
    order = np.argsort(batch.pos, kind="stable")
    batch = batch.select(order)
    return dict(name=f"deep_{n_sites}x{depth}", contigs=[("chr1", L, ref.tobytes(), 0)], batch=batch,
                regions=[(0, int(s) + 1, int(s) + 1) for s in sites], site_list=True,
                lib_names=[f"lib{i}" for i in range(n_libs)])


def testbam_case(bad_rg=False):
    """The reference's own fixture (R:test-data/test.bam + site_list), stored decoded under tests/golden/."""
    z = np.load(os.path.join(GOLDEN, "test_bam_bad_rg.npz" if bad_rg else "test_bam.npz"), allow_pickle=False)
    batch = ReadBatch(**{k: z[k] for k in ("tid", "pos", "flag", "mapq", "lib", "l_qseq", "nm", "sm", "cigar_off", "cigar",
                                           "seq_off", "seq", "qual_off", "qual")})
    win_beg = int(z["ref_win_beg"])
    ref = z["ref_win"].tobytes()
    return dict(name="test_bam_bad_rg" if bad_rg else "test_bam", contigs=[("21", int(z["chrom_len"]), ref, win_beg)],
                tid_map={20: 0}, batch=batch, regions=[(0, 10402985, 10402985), (0, 10405200, 10405200)], site_list=True,
                lib_names=[s for s in str(z["lib_names"]).split("\t") if s])


@functools.lru_cache(maxsize=None)
def testbam_chr21() -> bytes:
    """Contig 21 of test.bam as its ref.fa holds it: N everywhere except the window the fixture's reads touch."""
    z = np.load(os.path.join(GOLDEN, "test_bam.npz"))
    wb = int(z["ref_win_beg"])
    seq = np.full(int(z["chrom_len"]), ord("N"), dtype=np.uint8)
    seq[wb:wb + z["ref_win"].shape[0]] = z["ref_win"]
    return seq.tobytes()


def crafted_case(reads, regions, n_libs=1, L=300, seed=3):
    """A case from hand-placed reads: (pos, cigar, mismatch positions, library), optionally followed by mapq and flag (default
    60 and 0; SM is the mapq).  Every read copies the reference except at its mismatch positions."""
    rng = np.random.default_rng(seed)
    ref = bytes(rng.choice(list(b"ACGT"), L).astype(np.uint8))
    other = {ord("A"): "C", ord("C"): "G", ord("G"): "T", ord("T"): "A"}
    bb = BatchBuilder()
    for k, (pos, cigar, mism, lib, *rest) in enumerate(reads):
        mapq, flag = rest or (60, 0)
        seq, p = [], pos
        for n, op in re.findall(r"(\d+)([MID])", cigar):
            n = int(n)
            if op == "M":
                seq += [other[ref[q]] if q in mism else chr(ref[q]) for q in range(p, p + n)]
                p += n
            elif op == "D":
                p += n
            else:
                seq += ["A"] * n
        bb.add_sam(tid=0, pos=pos, flag=flag, mapq=mapq, lib=lib, cigar=cigar, seq="".join(seq), qual="I" * len(seq),
                   nm=len(mism), sm=mapq, qname=f"r{k}")
    b = bb.build()
    order = np.argsort(b.pos, kind="stable")
    return dict(name="crafted", contigs=[("chr1", L, ref, 0)], batch=b.select(order), regions=list(regions), site_list=False,
                lib_names=[f"lib{i}" for i in range(n_libs)])


def case_tid(case, ci):
    """BAM tid of contig index ci (the goldens' contig 21 has tid 20 in test.bam)."""
    inv = {v: k for k, v in case.get("tid_map", {}).items()}
    return inv.get(ci, ci)


def region_reads(case, ci, beg1, end1):
    """Records the index iterator yields for samfetch(d.beg-1, d.end) (R:bamreadcount.cpp:602)."""
    beg, end = beg1 - 1, end1
    tid = case_tid(case, ci)
    idx = case["batch"].fetch(tid, beg - 1, end)
    return tid, beg, end, case["batch"].select(idx)


class OracleRun(NamedTuple):
    text: str
    dump: str
    warnings: tuple


def run_oracle(case, flags, site_list=None) -> OracleRun:
    from oracle.oracle import Oracle
    sl = case["site_list"] if site_list is None else site_list
    o = Oracle(lib_names=case["lib_names"], **flags)
    for (ci, b1, e1) in case["regions"]:
        name, clen, seq, wb = case["contigs"][ci]
        tid, beg, end, sub = region_reads(case, ci, b1, e1)
        o.region(sub, tid=tid, beg=beg, end=end, contig=name, chrom_len=clen, ref_seq=seq, ref_win_beg=wb, site_list_mode=sl)
    return OracleRun(o.text(), o.dump(), o.warnings())


_ORACLE_RUNS: dict = {}


def run_oracle_cached(case, flags, site_list=None) -> OracleRun:
    """run_oracle, computed once per case name, flags and region mode (a case's name identifies it)."""
    sl = case["site_list"] if site_list is None else site_list
    key = (case["name"], tuple(sorted(flags.items())), sl)
    if key not in _ORACLE_RUNS:
        _ORACLE_RUNS[key] = run_oracle(case, flags, site_list=sl)
    return _ORACLE_RUNS[key]


@dataclasses.dataclass
class EngineRun:
    """What one brc_compute left: the text, the raw accumulator dump ("" when not asked for or under a site filter), the warning
    counters, the kernel launch count, the pool record count of packed() (-1 under a site filter) and, under a site filter, the
    selected sites."""
    text: str
    dump: str
    warnings: tuple
    launches: int
    n_sec: int
    selected: object = None


@contextlib.contextmanager
def open_engine(case, flags=None):
    """An engine with the case's libraries and the reference of every contig of the case."""
    from bam_readcount_b200.engine import Engine
    e = Engine(lib_names=case["lib_names"], **(flags or {}))
    try:
        for ci, (name, clen, seq, wb) in enumerate(case["contigs"]):
            e.set_reference(case_tid(case, ci), name, clen, seq, wb)
        yield e
    finally:
        e.close()


def push_regions(e, case, site_list, regions=None, push="one"):
    """begin_region / push / end_region for each region (default: the case's).  ``push``: "one" pushes a region's reads at
    once (borrowed by the engine), "halves" in two pushes (the engine copies them), a callable push(e, tid, beg, end, sub) as it
    likes.  Returns (tid, reads) per region."""
    pushed = []
    for (ci, b1, e1) in case["regions"] if regions is None else regions:
        tid, beg, end, sub = region_reads(case, ci, b1, e1)
        e.begin_region(tid, beg, end, site_list)
        if push == "one":
            e.push_reads(sub)
        elif push == "halves":
            h = sub.n_reads // 2
            e.push_reads(sub.select(np.arange(0, h)))
            e.push_reads(sub.select(np.arange(h, sub.n_reads)))
        else:
            push(e, tid, beg, end, sub)
        e.end_region()
        pushed.append((tid, sub))
    return pushed


def _compute(e, case, flags, pushed, dump) -> EngineRun:
    from bam_readcount_b200.engine import admitted
    res = e.compute()
    text = e.format_text(-1)
    d = ""
    if dump and res is not None and pushed:
        cnt = flags.get("max_cnt", 10_000_000)
        reads = ReadBatch.concat([sub.select(admitted(sub, tid, cnt)) for tid, sub in pushed])
        d = res.dump(reads, {case_tid(case, ci): (wb, seq) for ci, (_, _, seq, wb) in enumerate(case["contigs"])})
    return EngineRun(text=text, dump=d, warnings=e.warnings(), launches=e.launch_count(),
                     n_sec=e.packed().n_sec if res is not None else -1, selected=e.selected() if res is None else None)


def run_engine(case, flags, site_list=None, *, dump=True, site_filter=None, push="one") -> EngineRun:
    """The case's regions as one batch, one brc_compute.  site_filter: (min_alt_count, min_alt_fraction); push: push_regions."""
    sl = case["site_list"] if site_list is None else site_list
    with open_engine(case, flags) as e:
        if site_filter:
            e.set_site_filter(*site_filter)
        return _compute(e, case, flags, push_regions(e, case, sl, push=push), dump)


def run_engine_per_region(case, flags, site_list=None, *, dump=False) -> list:
    """One brc_compute per region with the deletion queue carried from one to the next (what brc-readcount does to bound its
    memory): an EngineRun per region, whose texts joined are the output."""
    sl = case["site_list"] if site_list is None else site_list
    with open_engine(case, flags) as e:
        e.set_queue_carry(True)
        runs = []
        for region in case["regions"]:
            e.reset()
            runs.append(_compute(e, case, flags, push_regions(e, case, sl, [region]), dump))
        e.set_queue_carry(False)
        return runs


def first_diff(got: str, want: str) -> str:
    """The first line where two texts differ, '' when they are equal (keeps pytest from diffing megabytes of text)."""
    if got == want:
        return ""
    la, lb = got.splitlines(), want.splitlines()
    for i, (x, y) in enumerate(zip(la, lb)):
        if x != y:
            return f"line {i}:\n got: {x[:300]}\nwant: {y[:300]}"
    return f"length differs: got {len(la)} lines, want {len(lb)}"


def assert_same(got: EngineRun, want: OracleRun, what: str = "", *, fields=("dump", "text", "warnings")):
    """The engine run equals the oracle's in the named fields (warnings: the engine's counters 0, 1 and 3, the oracle's three)."""
    pre = f"{what}: " if what else ""
    if "dump" in fields:
        assert got.dump == want.dump, pre + first_diff(got.dump, want.dump)
    if "text" in fields:
        assert got.text == want.text, pre + first_diff(got.text, want.text)
    if "warnings" in fields:
        w = got.warnings
        assert (w[0], w[1], w[3]) == want.warnings, f"{pre}warnings {w}, oracle {want.warnings}"


def region_geometry(case, region):
    """(tid, beg, end, reads, first_pos, n_slots, n_tiles) of one region as brc_begin_region / brc_end_region form them."""
    from kernel_model import kernel_constants
    tile = kernel_constants()["TILE"]
    tid, beg, end, sub = region_reads(case, *region)
    first_pos = max(beg - 1, 0)
    n_slots = max(0, min(end, int(sub.ref_end().max())) - first_pos) if sub.n_reads else 0
    return tid, beg, end, sub, first_pos, n_slots, (n_slots + tile - 1) // tile


_TORCH_VIEW = {np.dtype(np.uint16): np.int16, np.dtype(np.uint32): np.int32, np.dtype(np.uint64): np.int64}


def device_batch(batch, device, *, lead=None, cigar_pool=None):
    """The batch's arrays on the device: a CReadBatch of device pointers and the tensors that own them.  64 zero bytes follow
    the base and quality pools.  lead=("qual" or "seq", n): that pool starts n bytes into an allocation whose first n bytes are
    never written, its offsets shifted by n.  cigar_pool=(int32 tensor, n): the CIGAR ops are copied into the caller's tensor
    at op n, their offsets shifted by n."""
    import torch
    from bam_readcount_b200.engine import CReadBatch
    at = dict([lead]) if lead else {}
    pool = None
    if cigar_pool is not None:
        pool, at["cigar"] = cigar_pool
    keep = []

    def dev(a, pad=0, start=0, into=None):
        a = np.ascontiguousarray(a)
        a = torch.from_numpy(a.view(_TORCH_VIEW.get(a.dtype, a.dtype)))
        if into is None:
            into = torch.empty(start + a.shape[0] + pad, dtype=a.dtype, device=device)
            into[start + a.shape[0]:].zero_()
            keep.append(into)
        into[start:start + a.shape[0]].copy_(a)
        return into.data_ptr()

    def pool_at(name, pad=0, into=None):
        off = getattr(batch, name + "_off").astype(np.uint64) + np.uint64(at.get(name, 0))
        return [dev(off), dev(getattr(batch, name), pad, at.get(name, 0), into)]
    b = batch
    ptrs = [dev(b.tid), dev(b.pos), dev(b.flag), dev(b.mapq), dev(b.lib), dev(b.l_qseq), dev(b.nm), dev(b.sm)]
    ptrs += pool_at("cigar", into=pool) + pool_at("seq", 64) + pool_at("qual", 64)
    torch.cuda.synchronize(device)          # the engine reads them on a stream of its own
    return CReadBatch(b.n_reads, *ptrs), keep


def run_device(e, case, region, cbatch, stream, *, site_list=True, n_sec_cap=1 << 20) -> str:
    """One region of the case, its reads already on the device (device_batch), through brc_plan_device / brc_run_device /
    brc_fetch_device_results: the raw accumulator dump.  The device path admits every read it is given."""
    from bam_readcount_b200.engine import CRegion
    tid, beg, end, sub, first_pos, n_slots, _ = region_geometry(case, region)
    e.plan_device([CRegion(tid, beg, end, int(site_list), 0, sub.n_reads, 0, first_pos, n_slots)], sub.n_reads, n_sec_cap)
    e.run_device(cbatch, None, stream.cuda_stream)
    res = e.fetch_device_results(stream.cuda_stream)
    _, _, seq, wb = case["contigs"][region[0]]
    return res.dump(sub, {tid: (wb, seq)})


def assert_anchor(json_name: str, key: str, text: str):
    """The oracle's text hashes to what the unmodified reference binary printed (tests/golden/<json_name>, make_golden.py)."""
    with open(os.path.join(GOLDEN, json_name)) as fh:
        want = json.load(fh)[key]
    assert hashlib.sha256(text.encode("latin-1")).hexdigest() == want, f"{key}: oracle differs from the reference binary"


def cli() -> str:
    """Builds the engine library and brc-readcount; the path of brc-readcount."""
    from bam_readcount_b200 import build
    build.build()
    return build.build_cli()


def samtools() -> str:
    """The samtools the oracle build leaves in oracle/_ref; skips the test without it."""
    import pytest
    from oracle.oracle import REF_SAMTOOLS
    if not os.path.exists(REF_SAMTOOLS):
        pytest.skip("oracle/_ref/samtools not built")
    return REF_SAMTOOLS


def have_htslib() -> bool:
    """brc-readcount can be built with htslib, and so read CRAM: tools/build_htslib.sh has left its library."""
    return os.path.exists(os.path.join(ROOT, "bam_readcount_b200", "third_party", "htslib", "libhts.a"))


@functools.lru_cache(maxsize=None)
def _check_dir() -> str:
    d = tempfile.mkdtemp(prefix="brc_checks_")
    atexit.register(shutil.rmtree, d, True)
    return d


@functools.lru_cache(maxsize=None)
def check_program(name: str, *extra_flags: str) -> str:
    """Compiles tests/<name>.cpp, a CPU check program over headers in csrc/, once per test session; the executable's path.
    extra_flags follow the source on the g++ line (libraries to link, -pthread)."""
    exe = os.path.join(_check_dir(), name)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "bam_readcount_b200", "csrc"), "-o", exe,
                           os.path.join(ROOT, "tests", name + ".cpp"), *extra_flags])
    return exe


def write_fasta(path: str, contigs) -> str:
    """A FASTA of the (name, sequence bytes) contigs in 60 columns, and its .fai; the FASTA's path."""
    with open(path, "wb") as fa, open(path + ".fai", "w") as fai:
        off = 0
        for name, seq in contigs:
            head = f">{name}\n".encode()
            body = b"".join(seq[i:i + 60] + b"\n" for i in range(0, len(seq), 60))
            fa.write(head + body)
            fai.write(f"{name}\t{len(seq)}\t{off + len(head)}\t60\t61\n")
            off += len(head) + len(body)
    return path


def write_testbam_fasta(path: str) -> str:
    """The ref.fa of test.bam's contig 21 (testbam_chr21) at path, and its .fai; the path."""
    synth.write_fasta(path, "21", np.frombuffer(testbam_chr21(), dtype=np.uint8))
    return path


def sam_to_bam(sam: str, keep_sam: bool = True) -> str:
    """samtools view -b of a .sam file into the .bam beside it, indexed; the BAM's path.  Skips the test without samtools."""
    exe, bam = samtools(), sam[:-len(".sam")] + ".bam"
    subprocess.check_call([exe, "view", "-b", "-o", bam, sam])
    subprocess.check_call([exe, "index", bam])
    if not keep_sam:
        os.remove(sam)
    return bam


def write_bam(d: str, stem: str, batch, contigs, *, keep_sam: bool = True, **sam_kw) -> str:
    """The batch as d/<stem>.sam (synth.write_sam with the contigs [(name, length)] and sam_kw), then as an indexed
    d/<stem>.bam; the BAM's path."""
    sam = os.path.join(d, stem + ".sam")
    synth.write_sam(sam, batch, contigs, **sam_kw)
    return sam_to_bam(sam, keep_sam)


CONTIGS = {"chrA": (24000, 11), "chrB": (16000, 12), "chrC": (12000, 13)}       # name -> (length, reference seed)


def synthetic_bam(d, name, order, n_libs, seed, depth=8, no_nm=0) -> str:
    """A coordinate-sorted BAM d/<name>.bam whose @SQ lines are `order` (a subset of CONTIGS, in any order), with n_libs
    libraries (0: no @RG at all) and `no_nm` reads without an NM tag (they draw warnings)."""
    parts = []
    for tid, c in enumerate(order):
        ref = synth.synth_reference(CONTIGS[c][0], CONTIGS[c][1])
        parts.append(synth.synth_reads(ref, depth, seed=seed + 101 * tid, n_libs=max(n_libs, 1), tid=tid))
    b = ReadBatch.concat(parts)
    if no_nm:
        nm = np.array(b.nm, copy=True)
        nm[np.random.default_rng(seed).choice(b.n_reads, no_nm, replace=False)] = TAG_ABSENT
        b = dataclasses.replace(b, nm=nm)
    return write_bam(d, name, b, [(c, CONTIGS[c][0]) for c in order], keep_sam=False, n_libs=max(n_libs, 1),
                     read_group=n_libs > 0)


def load_golden_text(name: str) -> str:
    p = os.path.join(GOLDEN, name)
    if os.path.exists(p + ".gz"):
        with gzip.open(p + ".gz", "rb") as fh:
            return fh.read().decode("latin-1")
    with open(p, "rb") as fh:
        return fh.read().decode("latin-1")


def golden_texts():
    """[(name, text)] of every committed output text: the expected_* files and the *.txt.gz files, by name."""
    names = sorted({f[:-3] if f.endswith(".gz") else f for f in os.listdir(GOLDEN) if f.endswith(".txt.gz") or f.startswith("expected_")})
    return [(n, load_golden_text(n)) for n in names]
