"""The alternative-allele site filter (brc_set_site_filter, brc-readcount --min-alt-count / --min-alt-fraction).

The rule is defined on the text: ``select_lines`` below parses bam-readcount's line grammar (with -p library blocks) and keeps a
line iff one of its entries is an alternative allele with count >= min_alt_count and count >= min_alt_fraction * depth.  It is
the oracle: the filtered output of the engine must equal select_lines(unfiltered output) byte for byte.
CPU: select_lines on the committed goldens and on hand-written lines, CLI option validation, the exported symbols.
GPU: the engine and the C++ host, filtered, against select_lines of the reference goldens, the oracle and the unfiltered run.
"""
import os
import re
import subprocess

import numpy as np
import pytest

import cases
import golden_jobs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

_ENTRY = re.compile(r"^([=ACGTN]|[+-][^:]*):(\d+):")
_NT16 = {"A": 1, "C": 2, "G": 4, "T": 8}


def _line_entries(fields):
    """(allele, count) of every allele entry of a line's fields after the depth column (library names and braces skipped)."""
    for f in fields:
        m = _ENTRY.match(f)
        if m:
            yield m.group(1), int(m.group(2))


def is_alt(allele: str, ref_base: str) -> bool:
    if allele[0] in "+-":
        return True
    if allele not in _NT16:
        return False                          # "=" and "N"
    return _NT16[allele] != _NT16.get(ref_base.upper(), 15)


def line_passes(line: str, min_alt_count: int, min_alt_fraction: float, ref_lookup=None) -> bool:
    f = line.split("\t")
    ref = ref_lookup(f[0], int(f[1])) if ref_lookup else f[2]
    depth = int(f[3])
    return any(is_alt(a, ref) and c >= min_alt_count and float(c) >= min_alt_fraction * float(depth) for a, c in _line_entries(f[4:]))


def select_lines(text: str, min_alt_count: int, min_alt_fraction: float = 0.0, ref_lookup=None) -> str:
    """The lines of bam-readcount output `text` a site filter keeps.  ref_lookup(chrom, pos1) -> reference character; by
    default the line's own reference column."""
    return "".join(ln + "\n" for ln in text.splitlines() if line_passes(ln, min_alt_count, min_alt_fraction, ref_lookup))


THRESHOLDS = [(1, 0.0), (2, 0.05), (1, 0.2), (10 ** 6, 0.0)]


def _same(got: str, want: str) -> str:
    """'' when equal, else the first differing line (keeps pytest from diffing megabytes of text)."""
    if got == want:
        return ""
    for i, (x, y) in enumerate(zip(got.splitlines(), want.splitlines())):
        if x != y:
            return f"line {i}:\n got: {x[:300]}\nwant: {y[:300]}"
    return f"length differs: got {len(got.splitlines())} lines, want {len(want.splitlines())}"


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
def _golden_texts():
    names = sorted({f[:-3] if f.endswith(".gz") else f for f in os.listdir(GOLDEN) if f.endswith(".txt.gz") or f.startswith("expected_")})
    return [(n, cases.load_golden_text(n)) for n in names]


def test_select_lines_on_goldens_is_a_subsequence_dropping_only_lines_without_a_qualifying_allele():
    texts = _golden_texts()
    assert len(texts) >= 30
    for name, text in texts:
        lines = text.splitlines()
        for mc, mf in THRESHOLDS:
            kept = select_lines(text, mc, mf).splitlines()
            it = iter(lines)
            assert all(any(k == x for x in it) for k in kept), name           # an order-preserving subsequence
            keep = set(kept)
            for ln in lines:
                f = ln.split("\t")
                ok = [(a, c) for a, c in _line_entries(f[4:]) if is_alt(a, f[2]) and c >= mc and c >= mf * int(f[3])]
                assert (ln in keep) == bool(ok), (name, ln[:120])
        if len(lines) > 20:
            n1 = len(select_lines(text, 1).splitlines())
            assert 0 < n1 <= len(lines) and len(select_lines(text, 10 ** 6).splitlines()) == 0


_Z = "0.00:0.00:0.00:0:0:0.00:0.00:0.00:0:0.00:0.00:0.00"


def _e(allele, n):
    return f"{allele}:{n}:{_Z}"


def test_select_lines_hand_written_reference_bases_deletions_and_library_blocks():
    def line(ref, depth, *entries, libs=None):
        if libs:
            body = "".join(f"\t{lib}\t{{\t" + "\t".join(ents) + "\t}" for lib, ents in libs)
        else:
            body = "\t" + "\t".join(entries)
        return f"chr1\t100\t{ref}\t{depth}{body}"
    ref_only = [_e("=", 0), _e("A", 9), _e("C", 0), _e("G", 0), _e("T", 0), _e("N", 0)]
    assert not line_passes(line("A", 9, *ref_only), 1, 0.0)
    assert not line_passes(line("a", 9, *ref_only), 1, 0.0)                  # lower case: the same base
    assert line_passes(line("N", 9, *ref_only), 1, 0.0)                      # N: every base is alternative
    assert line_passes(line("R", 9, *ref_only), 1, 0.0)                      # IUPAC A/G: not exactly one base
    assert line_passes(line("C", 9, *ref_only), 9, 1.0)
    assert not line_passes(line("C", 10, *ref_only), 9, 1.0)                 # 9 < 1.0 * 10
    only_n = [_e("=", 3), _e("A", 0), _e("C", 0), _e("G", 0), _e("T", 0), _e("N", 7)]
    assert not line_passes(line("N", 10, *only_n), 1, 0.0)                   # "=" and "N" never are
    dels = [_e("=", 0), _e("A", 0), _e("C", 0), _e("G", 0), _e("T", 0), _e("N", 0), _e("-AC", 2)]
    assert line_passes(line("A", 2, *dels), 2, 1.0)                          # deletion-only site: the deletions count toward depth
    assert not line_passes(line("A", 2, *dels), 3, 0.0)
    ins = ref_only + [_e("+GT", 4)]
    assert line_passes(line("A", 13, *ins), 4, 0.3) and not line_passes(line("A", 13, *ins), 4, 0.31)
    per_lib = line("G", 12, libs=[("lib0", [_e("=", 0), _e("A", 0), _e("C", 0), _e("G", 6), _e("T", 0), _e("N", 0)]),
                                   ("lib1", [_e("=", 0), _e("A", 0), _e("C", 0), _e("G", 3), _e("T", 3), _e("N", 0)])])
    assert line_passes(per_lib, 3, 0.25) and not line_passes(per_lib, 4, 0.0) and not line_passes(per_lib, 3, 0.26)
    text = "\n".join([line("A", 9, *ref_only), per_lib, line("N", 9, *ref_only)]) + "\n"
    assert select_lines(text, 3) == per_lib + "\n" + line("N", 9, *ref_only) + "\n"
    assert select_lines(text, 1, ref_lookup=lambda c, p: "T") == text       # every A/G count is alternative to a T


def _cli():
    from bam_readcount_b200 import build
    build.build()
    return build.build_cli()


def test_cli_site_filter_option_validation():
    exe = _cli()
    bam = os.path.join(GOLDEN, "test.bam")
    env = dict(os.environ, BRC_CLI_DECODE_ONLY="1")
    for bad, msg in ((["--min-alt-count", "0"], b"--min-alt-count"), (["--min-alt-count", "x"], b"--min-alt-count"),
                     (["--min-alt-count", "3.5"], b"--min-alt-count"), (["--min-alt-fraction", "1.5"], b"--min-alt-fraction"),
                     (["--min-alt-fraction", "-0.1"], b"--min-alt-fraction"), (["--min-alt-fraction", "nan"], b"--min-alt-fraction"),
                     (["--min-alt-fraction", ""], b"--min-alt-fraction")):
        p = subprocess.run([exe] + bad + [bam, "21:10402985-10402990"], capture_output=True, env=env)
        assert p.returncode == 1 and msg in p.stderr, (bad, p.stderr)
    for good in (["--min-alt-count", "2"], ["--min-alt-fraction", "0.25"], ["--min-alt-count", "1", "--min-alt-fraction", "1"]):
        p = subprocess.run([exe] + good + [bam, "21:10402985-10402990"], capture_output=True, env=env)
        assert p.returncode == 0, (good, p.stderr)
    p = subprocess.run([exe, "-h"], capture_output=True)
    assert b"--min-alt-count N" in p.stdout and b"--min-alt-fraction F" in p.stdout


def test_site_filter_symbols_are_exported():
    from bam_readcount_b200 import build, engine
    build.build()
    lib = engine.load_library()
    for s in ("brc_set_site_filter", "brc_get_selected_results"):
        assert hasattr(lib, s) and s in engine.EXPORTS
    assert lib.brc_abi_version() == 2


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
def _run(case, flags, site_list, filt=None, want_selected=False):
    """cases.run_engine with an optional site filter: (text, selected results or None, regions, launch count)."""
    from bam_readcount_b200.engine import Engine
    e = Engine(lib_names=case["lib_names"], **flags)
    try:
        for ci, (name, clen, seq, wb) in enumerate(case["contigs"]):
            e.set_reference(cases.case_tid(case, ci), name, clen, seq, wb)
        if filt:
            e.set_site_filter(*filt)
        for (ci, b1, e1) in case["regions"]:
            tid, beg, end, sub = cases.region_reads(case, ci, b1, e1)
            e.begin_region(tid, beg, end, site_list)
            e.push_reads(sub)
            e.end_region()
        e.compute()
        text = e.format_text(-1)
        sel = e.selected() if (filt and want_selected) else None
        return text, sel, e.launch_count()
    finally:
        e.close()


_JOBS = [j for j in golden_jobs.jobs() if j[0].startswith(("syn-", "deep-", "edge-fuzz", "testbam-"))]


@pytest.mark.gpu
@pytest.mark.parametrize("job", _JOBS, ids=[j[0] for j in _JOBS])
def test_engine_filtered_text_equals_selected_golden(job):
    _, getter, flags, site_list, golden = job
    case = getter()
    want_all = cases.load_golden_text(golden)
    for mc, mf in THRESHOLDS:
        text, _, _ = _run(case, flags, site_list, (mc, mf))
        d = _same(text, select_lines(want_all, mc, mf))
        assert not d, (mc, mf, d)


@pytest.mark.gpu
@pytest.mark.parametrize("job", [j for j in _JOBS if j[3] or j[0].startswith("syn-")], ids=lambda j: j[0])
def test_device_selection_is_exact_without_carried_deletions(job):
    """Site lists and single argv regions carry no deletion from another region: the device's emit == 1 sites are exactly the
    lines the rule keeps (no superset slack)."""
    _, getter, flags, site_list, golden = job
    case = getter()
    want_all = cases.load_golden_text(golden)
    from bam_readcount_b200.engine import Engine
    for mc, mf in ((1, 0.0), (2, 0.05)):
        e = Engine(lib_names=case["lib_names"], **flags)
        try:
            for ci, (name, clen, seq, wb) in enumerate(case["contigs"]):
                e.set_reference(cases.case_tid(case, ci), name, clen, seq, wb)
            e.set_site_filter(mc, mf)
            for (ci, b1, e1) in case["regions"]:
                tid, beg, end, sub = cases.region_reads(case, ci, b1, e1)
                e.begin_region(tid, beg, end, site_list)
                e.push_reads(sub)
                e.end_region()
            e.compute()
            sel = e.selected()
            r = [p + 1 for p in sel.positions(1)]
            kept = [int(ln.split("\t")[1]) for ln in select_lines(want_all, mc, mf).splitlines()]
            assert r == kept, (mc, mf)
            assert not (sel.emit == 2).any() or not site_list       # keep-all ranges only follow argv regions
            # kept sites and their left neighbours; per argv region and library row, its last live site and that site's neighbour
            assert sel.n_sites <= 2 * len(kept) + 2 * sel.n_rows * len(case["regions"])
        finally:
            e.close()


@pytest.mark.gpu
def test_synthetic_whole_region_and_filter_off_is_unchanged():
    """cases.synthetic_case whole-region runs against select_lines of the oracle; after clear_site_filter the launches and the
    text are those of an engine that never had a filter."""
    case = cases.synthetic_case(L=40000, depth=30, seed=23, regions=((0, 1, 40000),), site_list=False)
    for flags in (dict(), dict(per_lib=True, insertion_centric=True), dict(min_mapq=20, min_bq=20)):
        want, _, _ = cases.run_oracle(case, flags, site_list=False)
        for mc, mf in THRESHOLDS:
            text, sel, _ = _run(case, flags, False, (mc, mf), want_selected=True)
            d = _same(text, select_lines(want, mc, mf))
            assert not d, (flags, mc, mf, d)
    fresh_text, _, fresh_launches = _run(case, dict(), False)
    from bam_readcount_b200.engine import BrcError, Engine
    name, clen, seq, wb = case["contigs"][0]
    e = Engine(lib_names=case["lib_names"])
    try:
        e.set_reference(0, name, clen, seq, wb)

        def step():
            e.reset()
            tid, beg, end, sub = cases.region_reads(case, 0, 1, 40000)
            e.begin_region(tid, beg, end, False)
            e.push_reads(sub)
            e.end_region()
            return e.compute()
        e.set_site_filter(2, 0.05)
        assert step() is None
        with pytest.raises(BrcError):
            e.packed()
        assert e.stage_ms(3) > 0.0
        e.clear_site_filter()
        res = step()
        assert res is not None and e.launch_count() == fresh_launches
        d = _same(e.format_text(-1), fresh_text)
        assert not d, d
        with pytest.raises(BrcError):
            e.selected()
        with pytest.raises(BrcError):
            e.set_site_filter(0)
        with pytest.raises(BrcError):
            e.set_site_filter(1, 1.5)
    finally:
        e.close()


def _write_ref(tmp):
    z = np.load(os.path.join(GOLDEN, "test_bam.npz"))
    L, wb = int(z["chrom_len"]), int(z["ref_win_beg"])
    seq = np.full(L, ord("N"), dtype=np.uint8)
    seq[wb:wb + z["ref_win"].shape[0]] = z["ref_win"]
    from bam_readcount_b200 import synth
    synth.write_fasta(os.path.join(tmp, "ref.fa"), "21", seq)
    return os.path.join(tmp, "ref.fa")


def _cli_pair(exe, argv, env=None, filt=(("--min-alt-count", "2"), ("--min-alt-fraction", "0.05"))):
    env = dict(os.environ, **(env or {}))
    full = subprocess.run([exe] + argv, capture_output=True, env=env)
    assert full.returncode == 0, full.stderr.decode()[-2000:]
    out = {}
    for fl in filt:
        p = subprocess.run([exe] + list(fl) + argv, capture_output=True, env=env)
        assert p.returncode == 0, p.stderr.decode()[-2000:]
        out[fl] = p
    return full, out


def _check_cli(exe, argv, env=None):
    filts = ((("--min-alt-count", "1"), 1, 0.0), (("--min-alt-count", "2", "--min-alt-fraction", "0.05"), 2, 0.05),
             (("--min-alt-fraction", "0.2"), 1, 0.2), (("--min-alt-count", "1000000"), 10 ** 6, 0.0))
    full, outs = _cli_pair(exe, argv, env, tuple(f for f, _, _ in filts))
    text = full.stdout.decode("latin-1")
    for fl, mc, mf in filts:
        p = outs[fl]
        d = _same(p.stdout.decode("latin-1"), select_lines(text, mc, mf))
        assert not d, (argv, fl, d)
        assert p.stderr == full.stderr                 # warning lines and counts do not depend on the filter
    return text


@pytest.mark.gpu
def test_cli_filtered_output_on_the_reference_fixture(tmp_path):
    """Site list, argv regions that overlap and that abut (deletions carried from one argv region into the next), -d."""
    exe = _cli()
    ref = _write_ref(str(tmp_path))
    bam = os.path.join(GOLDEN, "test.bam")
    sl = os.path.join(GOLDEN, "site_list")
    _check_cli(exe, ["-w", "0", "-f", ref, "-l", sl, bam])
    _check_cli(exe, ["-w", "0", "-p", "-f", ref, "-l", sl, bam])
    t = _check_cli(exe, ["-w", "0", "-f", ref, bam, "21:10402700-10403100", "21:10402950-10403300", "21:10403301-10403600", "21:10403550-10403700"])
    assert len(t.splitlines()) > 500
    _check_cli(exe, ["-w", "0", "-i", "-p", "-f", ref, bam, "21:10405000-10405300", "21:10405301-10405400", "21:10405100-10405200"])
    _check_cli(exe, ["-w", "0", "-d", "3", "-f", ref, bam, "21:10402700-10403100", "21:10403000-10403300"])


@pytest.mark.gpu
def test_cli_filtered_output_on_a_synthetic_bam(tmp_path):
    """A few tens of kb of synthetic BAM: one argv region cut into 3777-site windows (deletions across window edges), the
    device BGZF decode path, overlapping argv regions on it and a site list."""
    from oracle.oracle import REF_SAMTOOLS
    if not os.path.exists(REF_SAMTOOLS):
        pytest.skip("oracle/_ref/samtools not built")
    from bam_readcount_b200 import synth
    exe = _cli()
    case = cases.synthetic_case(L=40000, depth=30, seed=47, regions=((0, 1, 40000),), site_list=False)
    name, L, seq, _ = case["contigs"][0]
    d = str(tmp_path)
    synth.write_fasta(os.path.join(d, "ref.fa"), name, np.frombuffer(seq, dtype=np.uint8))
    synth.write_sam(os.path.join(d, "s.sam"), case["batch"], [(name, L)], n_libs=len(case["lib_names"]))
    subprocess.check_call([REF_SAMTOOLS, "view", "-b", "-o", os.path.join(d, "s.bam"), os.path.join(d, "s.sam")])
    subprocess.check_call([REF_SAMTOOLS, "index", os.path.join(d, "s.bam")])
    base = ["-w", "0", "-f", os.path.join(d, "ref.fa"), os.path.join(d, "s.bam")]
    want, _, _ = cases.run_oracle(case, dict(per_lib=True), site_list=False)
    t = _check_cli(exe, ["-p"] + base + ["chr1:1-40000"], env={"BRC_CLI_WINDOW": "3777"})
    diff = _same(t, want)
    assert not diff, diff
    _check_cli(exe, ["-i"] + base + ["chr1:1-40000"], env={"BRC_CLI_DEVICE_DECODE": "1"})
    _check_cli(exe, base + ["chr1:1001-9000", "chr1:8000-15000", "chr1:15001-20000", "chr1:100-300"])
    sl = tmp_path / "sites"
    sl.write_text("".join(f"chr1\t{s}\t{s + w}\n" for s, w in ((500, 40), (520, 10), (3000, 0), (9000, 300), (39000, 999))))
    _check_cli(exe, ["-w", "0", "-q", "20", "-b", "20", "-f", os.path.join(d, "ref.fa"), "-l", str(sl), os.path.join(d, "s.bam")])


# ---- crafted inputs for the deletion queue ------------------------------------------------------------------------------
def _crafted(reads, regions, n_libs=1, L=300, seed=3):
    """A case from hand-placed reads: (pos, cigar, mismatch positions, library).  Every read copies the reference except at
    its mismatch positions."""
    from bam_readcount_b200.batch import BatchBuilder
    rng = np.random.default_rng(seed)
    ref = bytes(rng.choice(list(b"ACGT"), L).astype(np.uint8))
    other = {ord("A"): "C", ord("C"): "G", ord("G"): "T", ord("T"): "A"}
    bb = BatchBuilder()
    for k, (pos, cigar, mism, lib) in enumerate(reads):
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
        bb.add_sam(tid=0, pos=pos, flag=0, mapq=60, lib=lib, cigar=cigar, seq="".join(seq), qual="I" * len(seq),
                   nm=len(mism), sm=60, qname=f"r{k}")
    b = bb.build()
    order = np.argsort(b.pos, kind="stable")
    return dict(name="crafted", contigs=[("chr1", L, ref, 0)], batch=b.select(order), regions=list(regions), site_list=False,
                lib_names=[f"lib{i}" for i in range(n_libs)])


@pytest.mark.gpu
def test_last_site_of_an_argv_region_keeps_the_deletion_from_its_left_neighbour():
    """The last site of an argv region is formed as a line even when it fails the rule; its left neighbour must be replayed, or
    the line loses the deletion queued there (and that deletion's share of the depth) and can pass a fraction it fails."""
    reads = [(40, "60M", {79} if k < 6 else set(), 0) for k in range(30)] + [(40, "39M1D20M", set(), 0)]
    case = _crafted(reads, [(0, 51, 80)])
    want, _, _ = cases.run_oracle(case, dict(), site_list=False)
    last = want.splitlines()[-1].split("\t")
    assert last[1] == "80" and any(f.startswith("-") for f in last[4:])          # the last line prints the deletion
    fractions = sorted({6 / 32, 6 / 31, 6 / 30, 0.19, 0.194, 0.195, 0.198, 0.2, 0.21} | {round(x, 3) for x in np.linspace(0.15, 0.25, 21)})
    for f in fractions:
        text, sel, _ = _run(case, dict(), False, (1, f), want_selected=True)
        diff = _same(text, select_lines(want, 1, f))
        assert not diff, (f, diff)


@pytest.mark.gpu
def test_per_library_queue_handed_to_an_overlapping_argv_region_is_the_unfiltered_one():
    """-p, two argv regions, the second inside the first.  Library 1's reads end before the first region does, and its line 61
    passes at count 2 while line 62, which prints library 1's deletion queued at 61, does not: that deletion must be consumed
    inside the first region, as the unfiltered pass does, and not print a second time in the second region."""
    reads = [(30, "80M", set(), 0) for _ in range(10)]
    reads += [(30, "40M", {60} if k < 3 else set(), 1) for k in range(5)] + [(30, "31M1D8M", set(), 1)]
    case = _crafted(reads, [(0, 41, 90), (0, 55, 65)], n_libs=2)
    flags = dict(per_lib=True)
    want, _, _ = cases.run_oracle(case, flags, site_list=False)
    for mc, mf in THRESHOLDS + [(2, 0.0), (3, 0.0)]:
        text, _, _ = _run(case, flags, False, (mc, mf))
        diff = _same(text, select_lines(want, mc, mf))
        assert not diff, (mc, mf, diff)
    lines62 = [ln for ln in want.splitlines() if ln.split("\t")[1] == "62"]
    assert len(lines62) == 2 and all(sum(f.startswith("-") for f in ln.split("\t")) == 1 for ln in lines62)
    assert [ln.split("\t")[1] for ln in select_lines(want, 2).splitlines()] == ["61", "61"]


@pytest.mark.gpu
def test_per_library_deletion_carried_through_a_region_that_drops_it():
    """-p, argv regions Z, A, B = Z again.  Z leaves library 1's deletion (printing at 61) in the queue; A starts after 61, so the
    unfiltered pass drops it at A's first line with library 1 reads, although no line of A passes.  B must then print its own
    copy of that deletion once, not twice."""
    reads = [(30, "100M", {60} if k < 3 else set(), 0) for k in range(20)]
    reads += [(30, "50M", set(), 1) for _ in range(5)] + [(30, "30M1D19M", set(), 1)]
    case = _crafted(reads, [(0, 41, 60), (0, 71, 120), (0, 41, 61)], n_libs=2)
    flags = dict(per_lib=True)
    want, _, _ = cases.run_oracle(case, flags, site_list=False)
    line61 = [ln for ln in want.splitlines() if ln.split("\t")[1] == "61"]
    assert len(line61) == 1 and sum(f.startswith("-") for f in line61[0].split("\t")) == 1
    for mc, mf in THRESHOLDS + [(2, 0.0), (3, 0.0)]:
        text, _, _ = _run(case, flags, False, (mc, mf))
        diff = _same(text, select_lines(want, mc, mf))
        assert not diff, (mc, mf, diff)


@pytest.mark.gpu
def test_device_only_reference_is_judged_by_the_printed_reference_column():
    """A contig set only on the device prints N as the reference base, so every base counts as alternative: the filtered text is
    still select_lines of the unfiltered text."""
    import torch
    from bam_readcount_b200.engine import Engine
    case = cases.synthetic_case(L=6000, depth=30, seed=5, regions=((0, 500, 5500),), site_list=False)
    name, clen, seq, wb = case["contigs"][0]
    dev = torch.tensor(np.frombuffer(seq + b"\0" * 64, dtype=np.uint8), device="cuda")
    torch.cuda.synchronize()
    texts = []
    for filt in (None, (20, 0.5)):
        e = Engine(lib_names=case["lib_names"])
        try:
            e.set_reference_device(0, name, clen, 0, dev.data_ptr(), len(seq), torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
            if filt:
                e.set_site_filter(*filt)
            tid, beg, end, sub = cases.region_reads(case, 0, 500, 5500)
            e.begin_region(tid, beg, end, False)
            e.push_reads(sub)
            e.end_region()
            e.compute()
            texts.append(e.format_text(-1))
        finally:
            e.close()
    full, filtered = texts
    assert all(ln.split("\t")[2] == "N" for ln in full.splitlines()[:50])
    kept = select_lines(full, 20, 0.5)
    assert len(kept.splitlines()) > 1000
    diff = _same(filtered, kept)
    assert not diff, diff
