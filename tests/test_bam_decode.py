"""BAM record decoding against htslib's rules, on hand-made files (tests/bam_craft.py).

Every BAM decoder here -- the device kernels of brc_bgzf.cu, brc-readcount's host reader, bamio.read_bam -- must read a record's
NM, SM, RG and CIGAR the way the reference binary does: the first tag of each name, a `d` value skipped as 8 bytes, a non-integer
NM/SM present and worth 0, the first RG whatever its type, and a long CIGAR stored in CG:B:I behind a <l_qseq>S placeholder.
bam_craft.Restated states those rules independently; tests/golden/decode_sha256.json pins its results to the reference binary.

CPU: the oracle on the restatement's reads prints what the reference printed (stdout hashes); bamio equals the restatement; the
DEFLATE core (brc_bgzf.cuh) inflates the crafted members as zlib does; the DEFLATE encoder's audit (tests/deflate_craft.py)
covers every construct.  GPU: the device-decoded batch equals the restatement field for field over differently cut and
compressed copies of every file, the hand-built DEFLATE members and hand-made spans; brc_push_bam_span, brc_push_reads and the
oracle agree; brc-readcount prints the reference's stdout and stderr, with host decode, device decode and on CRAM."""
import hashlib
import json
import os
import subprocess
import zlib

import numpy as np
import pytest

import bam_craft
import cases
from bam_readcount_b200 import bamio
from oracle.oracle import REF_SAMTOOLS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
FLAGS = {"default": {}, "p": dict(per_lib=True), "i": dict(insertion_centric=True), "q20b20": dict(min_mapq=20, min_bq=20)}
ARRAYS = ("pos", "flag", "mapq", "lib", "l_qseq", "nm", "sm", "cigar_off", "cigar", "seq_off", "seq", "qual_off", "qual")
NAMES = ["cg", "dtag", "nmtype", "rg", "rg_nolib", "trunc", "long"]


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    if not os.path.exists(REF_SAMTOOLS):
        pytest.skip("oracle/_ref/samtools not built")
    d = str(tmp_path_factory.mktemp("craft"))
    files = bam_craft.write_corpus(d, REF_SAMTOOLS)
    return {f["name"]: dict(f, restated=None if f["bam"].endswith(".cram") else bam_craft.Restated(f["bam"])) for f in files}


def _fasta_seq(path):
    with open(path) as fh:
        return fh.read().split("\n", 1)[1].replace("\n", "").encode()


def _case(f, batch):
    r = f["restated"]
    regs = [(0, int(x.split(":")[1].split("-")[0]), int(x.split("-")[1])) for x in f["regions"]]
    return dict(name=f["name"], contigs=[(r.refs[0][0], r.refs[0][1], _fasta_seq(f["fasta"]), 0)], batch=batch, regions=regs,
                site_list=False, lib_names=r.lib_name_strs)


def _assert_same_reads(got, want, what):
    assert got.n_reads == want.n_reads, what
    for k in ARRAYS:
        a, b = getattr(got, k), getattr(want, k)
        assert a.dtype == b.dtype and np.array_equal(a, b), f"{what}: {k} differs"


def _reference_sha():
    with open(os.path.join(GOLDEN, "decode_sha256.json")) as fh:
        return json.load(fh)


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------
def test_corpus_holds_every_rule(corpus):
    """The crafted reads reach each rule: a moved CG CIGAR (and a >65535-op one), a d tag, non-integer NM/SM, every integer NM
    type, a non-string first RG, an H-typed RG, an RG ID longer than 44 bytes, and unwalkable aux tails."""
    b = {k: f["restated"].batch for k, f in corpus.items() if f["restated"] is not None}
    n_cig = lambda x: np.diff(x.cigar_off.astype(np.int64))               # noqa: E731
    assert (n_cig(b["cg"])[:3] == 5).all() and (n_cig(b["cg"])[3:] == 2).all()
    assert n_cig(b["long"]).max() == 65537
    assert list(b["nmtype"].nm[:9]) == [0, 0, 0, 0, 0, 0, 5, 5, 0] and list(b["nmtype"].sm[6:8]) == [0, 0]
    assert list(b["nmtype"].nm[9:15]) == [-3, 200, -300, 60000, -5, 3000000000 - 2 ** 32]
    assert list(b["dtag"].nm) == [5, 2, 5] and b["dtag"].lib[0] == 1
    rg = corpus["rg"]["restated"]
    assert [rg.lib_name_strs[i] for i in b["rg"].lib] == ["L4", "L3", "L2"] and len(bam_craft.LONG_RG) > 44
    assert (b["rg_nolib"].lib[1:] == 0xFFFF).all() and b["rg_nolib"].lib[0] != 0xFFFF
    assert (b["trunc"].nm == np.int32(-2 ** 31)).tolist() == [True, True, True, False, True, False]
    assert b["trunc"].lib[3] == 0 and b["trunc"].lib[5] == 0xFFFF


@pytest.mark.parametrize("fname", list(FLAGS))
@pytest.mark.parametrize("name", [n for n in NAMES if n != "trunc"])
def test_restatement_is_what_the_reference_binary_reads(corpus, name, fname):
    """The oracle on the restatement's reads prints byte for byte what the unmodified reference binary printed."""
    text, _, _ = cases.run_oracle(_case(corpus[name], corpus[name]["restated"].batch), FLAGS[fname])
    assert hashlib.sha256(text.encode("latin-1")).hexdigest() == _reference_sha()[f"{name}_{fname}"]["stdout"]


@pytest.mark.parametrize("name", NAMES)
def test_bamio_equals_restatement(corpus, name):
    hdr, batch = bamio.read_bam(corpus[name]["bam"])
    r = corpus[name]["restated"]
    _assert_same_reads(batch, r.batch, name)
    assert hdr.lib_names == r.lib_name_strs


def _recut(f, how):
    """The records of f in new BGZF members: ("level", n), ("strategy", s), ("cut", n) n-byte members, ("empty",) an empty
    member between two halves, ("full",) 65536-byte members."""
    raw = bam_craft._gunzip_members(open(f["bam"], "rb").read())
    r = f["restated"]
    hdr_len = len(bam_craft.header_bytes(r.text, r.refs))
    data = raw[hdr_len:]
    kw = {}
    if how[0] == "level":
        kw["level"] = how[1]
    elif how[0] == "strategy":
        kw["strategy"] = how[1]
    elif how[0] == "cut":
        kw["members"] = lambda d: bam_craft.chunks_default(d, how[1])
    elif how[0] == "empty":
        kw["members"] = lambda d: bam_craft.chunks_default(d[:len(d) // 2]) + [b""] + bam_craft.chunks_default(d[len(d) // 2:])
    elif how[0] == "full":
        kw["members"] = lambda d: bam_craft.chunks_default(d, 65536)
        kw["level"] = 9
    out = f["bam"][:-4] + "_" + "_".join(map(str, how)) + ".bam"
    return bam_craft.write_bam(out, r.text, r.refs, [data], **kw)


RECUTS = [("level", 0), ("level", 1), ("level", 9), ("strategy", zlib.Z_FILTERED), ("strategy", zlib.Z_HUFFMAN_ONLY),
          ("strategy", zlib.Z_RLE), ("strategy", zlib.Z_FIXED), ("cut", 97), ("empty",), ("full",)]


def test_deflate_core_on_the_recut_corpus(corpus, tmp_path):
    """The DEFLATE core of the device kernel (one lane, on the CPU) against zlib on every member of every recut file, and its
    refusal of each member cut in half."""
    from test_bgzf_device import HARNESS
    src = os.path.join(str(tmp_path), "h.cpp")
    with open(src, "w") as fh:
        fh.write(HARNESS)
    exe = os.path.join(str(tmp_path), "h")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "bam_readcount_b200", "csrc"), "-o", exe, src, "-lz"])
    files = [_recut(corpus[n], how) for n in ("cg", "long") for how in RECUTS]
    nblk, bad = map(int, subprocess.check_output([exe] + files).split())
    assert bad == 0 and nblk > 100


@pytest.fixture(scope="module")
def crafted(tmp_path_factory):
    """deflate.bam (every crafted DEFLATE member inside one read's qualities) and frame.bam (two contigs, three members)."""
    d = str(tmp_path_factory.mktemp("deflate"))
    path, info = bam_craft.deflate_bam(d)
    fpath, starts, cuts = bam_craft.frame_bam(d)
    return dict(deflate=path, deflate_info=info, frame=fpath, starts=starts, cuts=[int(c) for c in cuts])


def test_deflate_corpus_covers_every_construct(crafted):
    """The encoder's audit: every construct the device decoder has a separate path or table for occurs in the crafted members,
    and the read carrying them spans three or more members."""
    import deflate_craft
    audit = deflate_craft.audit(deflate_craft.corpus_members())
    assert all(audit.values()), [k for k, v in audit.items() if not v]
    beg, end = crafted["deflate_info"][:2]
    assert sum(1 for e in crafted["deflate_info"][2:] if beg < e < end) >= 2


def test_deflate_core_on_the_crafted_members(crafted, tmp_path):
    """The DEFLATE core (one lane, on the CPU) against zlib on every crafted member, and its refusal of each member cut in half;
    bamio and the restatement read the same records from both crafted files."""
    from test_bgzf_device import HARNESS
    src = os.path.join(str(tmp_path), "h.cpp")
    with open(src, "w") as fh:
        fh.write(HARNESS)
    exe = os.path.join(str(tmp_path), "h")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "bam_readcount_b200", "csrc"), "-o", exe, src, "-lz"])
    nblk, bad = map(int, subprocess.check_output([exe, crafted["deflate"]]).split())
    assert bad == 0 and nblk >= 8
    for path in (crafted["deflate"], crafted["frame"]):
        _assert_same_reads(bamio.read_bam(path)[1], bam_craft.Restated(path).batch, path)


def _blocks(path):
    """(compressed offset relative to the first record member, isize) of every member after the header's, and that offset."""
    with open(path, "rb") as fh:
        d = fh.read()
    o = first = int.from_bytes(d[16:18], "little") + 1
    out = []
    while o + 18 <= len(d):
        bs = int.from_bytes(d[o + 16:o + 18], "little") + 1
        out.append((o - first, int.from_bytes(d[o + bs - 4:o + bs], "little")))
        o += bs
    return out, first


def frame_spans(crafted):
    """Hand-made spans over frame.bam: (entries, end_voff, first read, end read).  Entries in the middle of a member and at
    voff & 0xFFFF == isize of the member before (the same record start written the other way); end_voff inside or absent."""
    blocks, _ = _blocks(crafted["frame"])
    ustart = np.cumsum([0] + [b[1] for b in blocks])
    st = crafted["starts"]

    def voff(u):
        i = max(k for k in range(len(blocks)) if ustart[k] <= u and (u < ustart[k] + blocks[k][1] or k == len(blocks) - 1))
        return blocks[i][0] << 16 | (u - int(ustart[i]))

    def at_end_of_previous(u):
        i = [int(x) for x in ustart].index(u)
        assert i > 0
        return blocks[i - 1][0] << 16 | blocks[i - 1][1]
    assert voff(st[5]) & 0xFFFF and st[8] == crafted["cuts"][1]
    return [([voff(st[0]), voff(st[5]), at_end_of_previous(st[8])], voff(st[11]), 0, 11),
            ([voff(st[3])], -1, 3, 14),
            ([at_end_of_previous(st[8])], -1, 8, 14),
            ([voff(st[1]), voff(st[4])], at_end_of_previous(st[8]), 1, 8)]


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_device_inflates_the_crafted_members(crafted):
    """decode_bam_span on deflate.bam: 32 lanes per member over every crafted DEFLATE construct; all 13 arrays equal the
    restatement (the crafted bytes are one read's qualities)."""
    from bam_readcount_b200.engine import Engine
    r = bam_craft.Restated(crafted["deflate"])
    e = Engine(per_lib=True, lib_names=["x"] * 8)
    try:
        _assert_same_reads(e.decode_bam_span(_whole_span(crafted["deflate"], r)), r.batch, "deflate.bam")
    finally:
        e.close()


@pytest.mark.gpu
def test_device_framing_of_hand_made_spans(crafted):
    """Each hand-made span decodes to exactly the records between its first entry and its end, field for field; records of the
    other contig inside the span come back marked unmapped (never admitted)."""
    from bam_readcount_b200.engine import Engine
    r = bam_craft.Restated(crafted["frame"])
    _, first = _blocks(crafted["frame"])
    with open(crafted["frame"], "rb") as fh:
        comp = fh.read()[first:]
    e = Engine(per_lib=True, lib_names=["x"] * 8)
    try:
        for entries, end_voff, lo, hi in frame_spans(crafted):
            got = e.decode_bam_span(dict(comp=comp, entries=entries, end_voff=end_voff, tid=0, rg_lib=r.rg_lib()))
            want = r.batch.select(np.arange(lo, hi))
            want.flag = np.where(want.tid != 0, want.flag | 4, want.flag).astype(np.uint16)
            _assert_same_reads(got, want, (entries, end_voff))
    finally:
        e.close()

def _whole_span(path, restated):
    """Every record member of a crafted BAM as one span: the first record starts at virtual offset 0 of the first member after
    the header's."""
    with open(path, "rb") as fh:
        d = fh.read()
    hdr_end = int.from_bytes(d[16:18], "little") + 1
    return dict(comp=d[hdr_end:], entries=[0], end_voff=-1, tid=0, rg_lib=restated.rg_lib())


@pytest.mark.gpu
def test_device_decode_equals_restatement(corpus):
    """All 13 arrays of the device-decoded batch equal the restatement, for every crafted file and every recut of it (stored,
    fast, best, filtered, Huffman-only, RLE and fixed-Huffman members; 97-byte members, so records span many members; an empty
    member mid-span; 64 KiB members)."""
    from bam_readcount_b200.engine import Engine
    e = Engine(per_lib=True, lib_names=["x"] * 8)
    try:
        for name in NAMES:
            f = corpus[name]
            for path in [f["bam"]] + [_recut(f, how) for how in RECUTS]:
                got = e.decode_bam_span(_whole_span(path, f["restated"]))
                _assert_same_reads(got, f["restated"].batch, os.path.basename(path))
    finally:
        e.close()


def _engine_text(f, host, regions, span=False, flags=None):
    """Engine text over argv regions: the reads bamio decoded, or (one region only) the file's compressed span."""
    from bam_readcount_b200.engine import Engine
    r = f["restated"]
    case = _case(f, host)
    e = Engine(lib_names=case["lib_names"], **(flags or {}))
    try:
        name, clen, seq, wb = case["contigs"][0]
        e.set_reference(0, name, clen, seq, wb)
        for (_, b1, e1) in regions:
            tid, beg, end, sub = cases.region_reads(case, 0, b1, e1)
            e.begin_region(tid, beg, end, False)
            if span:
                e.push_bam_span(bamio.bam_span(f["bam"], bamio.BaiIndex(f["bam"] + ".bai"), 0, beg - 1, end, r.rg_lib()))
            else:
                e.push_reads(sub)
            e.end_region()
        e.compute()
        return e.format_text(-1)
    finally:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fname", list(FLAGS))
def test_reads_and_span_equal_the_reference(corpus, fname, monkeypatch):
    """brc_push_reads of bamio's reads prints the reference binary's stdout, and brc_push_bam_span (one span per region) prints
    what brc_push_reads prints for that region.  The long-CIGAR file also runs with the deep-site kernel forced, which puts a
    read of more than 65535 ops through K0/K1 and the deep path."""
    want = _reference_sha()
    for name in [n for n in NAMES if n != "trunc"]:
        f = corpus[name]
        _, host = bamio.read_bam(f["bam"])
        regions = _case(f, host)["regions"]
        for deep in ([False, True] if name == "long" else [False]):
            if deep:
                monkeypatch.setenv("BRC_DEEP_MIN_READS", "1")
            text = _engine_text(f, host, regions, flags=FLAGS[fname])
            assert hashlib.sha256(text.encode("latin-1")).hexdigest() == want[f"{name}_{fname}"]["stdout"], (name, deep)
            for reg in regions:
                assert _engine_text(f, host, [reg], span=True, flags=FLAGS[fname]) == _engine_text(f, host, [reg], flags=FLAGS[fname]), (name, reg, deep)
            monkeypatch.delenv("BRC_DEEP_MIN_READS", raising=False)
        # text, raw accumulators and warning counts: engine on bamio's reads == oracle on the restatement's reads
        etext, edump, ewarn, _ = cases.run_engine(_case(f, host), FLAGS[fname])
        otext, odump, owarn = cases.run_oracle(_case(f, f["restated"].batch), FLAGS[fname])
        assert (etext, edump) == (otext, odump) and (ewarn[0], ewarn[1], ewarn[3]) == owarn, name


@pytest.mark.gpu
@pytest.mark.parametrize("fname", list(FLAGS))
def test_cli_reads_unwalkable_aux_as_the_restatement_does(corpus, fname):
    """Row 5 and the unknown-type control through brc-readcount's own BAM reader: its stdout equals the engine's on the
    restatement's reads (the reference's own output differs there, see DESIGN.md §9), and device decode prints the same."""
    from bam_readcount_b200 import build
    exe = build.build_cli()
    f = corpus["trunc"]
    want, _, _, _ = cases.run_engine(_case(f, f["restated"].batch), FLAGS[fname])
    args = [exe, "-w", "0"] + bam_craft.FLAG_SETS[fname] + ["-f", f["fasta"], f["bam"]] + f["regions"]
    host = subprocess.run(args, capture_output=True)
    dev = subprocess.run(args, capture_output=True, env=dict(os.environ, BRC_CLI_DEVICE_DECODE="1"))
    assert host.returncode == 0 and dev.returncode == 0, host.stderr.decode()[-1500:]
    assert host.stdout.decode("latin-1") == want and dev.stdout == host.stdout


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rg_cram", "rg_nolib_cram"])
def test_cli_cram_reads_the_first_rg_whatever_its_type(corpus, name):
    """The RG files as CRAM, read through htslib: brc-readcount -p prints the reference's stdout and stderr on the same CRAM
    (an H-typed first RG names its read group; a non-string one leaves the read without a library)."""
    from bam_readcount_b200 import build
    if not os.path.exists(os.path.join(ROOT, "bam_readcount_b200", "third_party", "htslib", "libhts.a")):
        pytest.skip("host built without htslib (tools/build_htslib.sh)")
    exe = build.build_cli()
    f = corpus[name]
    p = subprocess.run([exe, "-w", "1", "-p", "-f", f["fasta"], f["bam"]] + f["regions"], capture_output=True)
    want = _reference_sha()[f"{name}_p"]
    assert p.returncode == 0, p.stderr.decode()[-1500:]
    assert hashlib.sha256(p.stdout).hexdigest() == want["stdout"] and hashlib.sha256(p.stderr).hexdigest() == want["stderr"]


@pytest.mark.gpu
@pytest.mark.parametrize("fname", list(FLAGS))
def test_cli_prints_what_the_reference_prints(corpus, fname):
    """brc-readcount -w 1 prints the reference's stdout and stderr (the NM/SM/library warnings) with host decode, and the same
    stdout with device decode."""
    from bam_readcount_b200 import build
    exe = build.build_cli()
    want = _reference_sha()
    for name in [n for n in NAMES if n != "trunc"]:
        f = corpus[name]
        args = [exe, "-w", "1"] + bam_craft.FLAG_SETS[fname] + ["-f", f["fasta"], f["bam"]] + f["regions"]
        host = subprocess.run(args, capture_output=True)
        dev = subprocess.run(args, capture_output=True, env=dict(os.environ, BRC_CLI_DEVICE_DECODE="1"))
        key = f"{name}_{fname}"
        assert host.returncode == 0 and dev.returncode == 0, dev.stderr.decode()[-1500:]
        assert hashlib.sha256(host.stdout).hexdigest() == want[key]["stdout"], key
        assert hashlib.sha256(host.stderr).hexdigest() == want[key]["stderr"], (key, host.stderr.decode()[-800:])
        assert dev.stdout == host.stdout, key
