"""Cohort mode of the C++ host: `brc-readcount --bam-list FILE` runs every sample of FILE in one process, and each sample's OUT
and ERR must hold exactly the bytes a run on that input alone prints on STDOUT and STDERR, with the same options and regions.
CPU tests use the decode-only hook (BRC_CLI_DECODE_ONLY: per-region record summaries instead of counts); GPU tests compare
the real output, flag set by flag set, and test.bam also against the reference's goldens."""
import concurrent.futures
import os
import shutil
import subprocess

import numpy as np
import pytest

import cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CRAM_DATA = os.path.join(ROOT, "oracle", "_ref", "test-data")
CONTIGS = {"chrA": (24000, 11), "chrB": (16000, 12), "chrC": (12000, 13)}       # name -> (length, reference seed)


def _cli():
    from bam_readcount_b200 import build
    build.build()
    return build.build_cli()


def _samtools():
    from oracle.oracle import REF_SAMTOOLS
    if not os.path.exists(REF_SAMTOOLS):
        pytest.skip("oracle/_ref/samtools not built")
    return REF_SAMTOOLS


def _have_htslib(exe):
    return os.path.exists(os.path.join(ROOT, "bam_readcount_b200", "third_party", "htslib", "libhts.a")) and \
        os.path.exists(os.path.join(CRAM_DATA, "twolib.sorted.cram"))


def _write_fasta(path, contigs):
    """Multi-contig FASTA (60 columns) and its .fai."""
    with open(path, "wb") as fa, open(path + ".fai", "w") as fai:
        off = 0
        for name, seq in contigs:
            head = f">{name}\n".encode()
            fa.write(head)
            off += len(head)
            body = b"".join(seq[i:i + 60] + b"\n" for i in range(0, len(seq), 60))
            fa.write(body)
            fai.write(f"{name}\t{len(seq)}\t{off}\t60\t61\n")
            off += len(body)


def _synthetic_bam(d, name, order, n_libs, seed, depth=8, no_nm=0):
    """A coordinate-sorted BAM whose @SQ lines are `order` (a subset of CONTIGS, in any order), with n_libs libraries
    (0: no @RG at all) and `no_nm` reads without an NM tag (they draw warnings)."""
    import dataclasses
    from bam_readcount_b200 import synth
    from bam_readcount_b200.batch import ReadBatch, TAG_ABSENT
    parts = []
    for tid, c in enumerate(order):
        ref = synth.synth_reference(CONTIGS[c][0], CONTIGS[c][1])
        parts.append(synth.synth_reads(ref, depth, seed=seed + 101 * tid, n_libs=max(n_libs, 1), tid=tid))
    b = ReadBatch.concat(parts)
    if no_nm:
        nm = np.array(b.nm, copy=True)
        nm[np.random.default_rng(seed).choice(b.n_reads, no_nm, replace=False)] = TAG_ABSENT
        b = dataclasses.replace(b, nm=nm)
    sam, bam = os.path.join(d, name + ".sam"), os.path.join(d, name + ".bam")
    synth.write_sam(sam, b, [(c, CONTIGS[c][0]) for c in order], n_libs=max(n_libs, 1), read_group=n_libs > 0)
    subprocess.check_call([_samtools(), "view", "-b", "-o", bam, sam])
    subprocess.check_call([_samtools(), "index", bam])
    os.remove(sam)
    return bam


@pytest.fixture(scope="module")
def cohort(tmp_path_factory):
    """Inputs of every test here: synthetic BAMs with 0, 2 and 5 libraries, different @SQ orders and contig subsets; the
    reference's test.bam and test_bad_rg.bam; test.bam cut inside a BGZF block; one FASTA holding every contig; a site list
    over all of them plus a contig no input has."""
    from bam_readcount_b200 import synth
    d = str(tmp_path_factory.mktemp("cohort"))
    s = {
        "syn5a": _synthetic_bam(d, "syn5a", ["chrA", "chrB", "chrC"], 5, seed=21, no_nm=60),
        "syn2": _synthetic_bam(d, "syn2", ["chrB", "chrA"], 2, seed=22),
        "syn5b": _synthetic_bam(d, "syn5b", ["chrC", "chrA", "chrB"], 5, seed=23),
        "syn0": _synthetic_bam(d, "syn0", ["chrA", "chrC"], 0, seed=24, no_nm=10),
        "test": os.path.join(GOLDEN, "test.bam"),
        "bad_rg": os.path.join(GOLDEN, "test_bad_rg.bam"),
    }
    cut = os.path.join(d, "cut.bam")
    with open(os.path.join(GOLDEN, "test.bam"), "rb") as fh:
        open(cut, "wb").write(fh.read()[:60000])
    shutil.copy(os.path.join(GOLDEN, "test.bam.bai"), cut + ".bai")
    s["cut"] = cut
    cram = os.path.join(CRAM_DATA, "twolib.sorted.cram")
    if os.path.exists(cram):                                    # the CRAM without its index, and with an index older than it
        s["cram_noidx"] = os.path.join(d, "noidx.cram")
        shutil.copy(cram, s["cram_noidx"])
        s["cram_old_idx"] = os.path.join(d, "old_idx.cram")
        shutil.copy(cram, s["cram_old_idx"])
        shutil.copy(cram + ".crai", s["cram_old_idx"] + ".crai")
        os.utime(s["cram_old_idx"] + ".crai", (1e9, 1e9))
    z = np.load(os.path.join(GOLDEN, "test_bam.npz"))
    chr21 = np.full(int(z["chrom_len"]), ord("N"), dtype=np.uint8)
    wb = int(z["ref_win_beg"])
    chr21[wb:wb + z["ref_win"].shape[0]] = z["ref_win"]
    rand1k = b"".join(open(os.path.join(GOLDEN, "rand1k.fa"), "rb").read().split(b"\n")[1:])
    fa = os.path.join(d, "all.fa")
    _write_fasta(fa, [("21", chr21.tobytes()), ("rand1k", rand1k)] +
                 [(c, synth.synth_reference(L, sd).tobytes()) for c, (L, sd) in CONTIGS.items()])
    rng = np.random.default_rng(4)
    lines = open(os.path.join(GOLDEN, "site_list")).read() + open(os.path.join(GOLDEN, "twolib_site_list.txt")).read()
    for c, (L, _) in CONTIGS.items():
        for p in np.sort(rng.integers(200, L - 400, 25)):
            lines += f"{c}\t{p}\t{p + int(rng.integers(0, 30))}\n"
    lines += "chrZ\t100\t200\n" + "chrB\t3000\t3400\n"
    sl = os.path.join(d, "sites")
    open(sl, "w").write(lines)
    return dict(dir=d, samples=s, fasta=fa, sites=sl)


def _single(exe, args, inp, regions, env):
    p = subprocess.run([exe] + args + [inp] + regions, capture_output=True, env=env)
    return p.returncode, p.stdout, p.stderr


def _run_cohort(exe, d, tag, args, inputs, regions, env, err_col=True):
    """One --bam-list run over `inputs`; returns (exit status, its STDERR, [(OUT bytes, ERR bytes)] per input)."""
    lst = os.path.join(d, f"{tag}.list")
    outs = [os.path.join(d, f"{tag}.{k}.out") for k in range(len(inputs))]
    errs = [os.path.join(d, f"{tag}.{k}.err") if err_col else o + ".log" for k, o in enumerate(outs)]
    with open(lst, "w") as fh:
        for k, inp in enumerate(inputs):
            fh.write(f"{inp}\t{outs[k]}" + (f"\t{errs[k]}" if err_col else "") + "\n")
            if k == 1:
                fh.write("\n")                                  # empty lines are skipped
    p = subprocess.run([exe] + args + ["--bam-list", lst] + regions, capture_output=True, env=env)
    return p.returncode, p.stderr, [(open(o, "rb").read(), open(e, "rb").read()) for o, e in zip(outs, errs)]


def _check_cohort_equals_single_runs(exe, d, tag, args, inputs, regions, env):
    rc, stderr, got = _run_cohort(exe, d, tag, args, inputs, regions, env)
    with concurrent.futures.ThreadPoolExecutor(4) as pool:
        want = list(pool.map(lambda inp: _single(exe, args, inp, regions, env), inputs))
    for inp, (o, e), (wrc, wo, we) in zip(inputs, got, want):
        assert o == wo, (tag, inp, "OUT")
        assert e == we, (tag, inp, "ERR")
    n_failed = sum(1 for w in want if w[0] != 0)
    assert rc == (1 if n_failed else 0), stderr.decode()
    assert len([ln for ln in stderr.decode().splitlines() if " failed" in ln]) == n_failed, stderr.decode()
    return got, want


# ---------------------------------------------------------------------------------------------------------------- CPU
DECODE_ONLY = dict(os.environ, BRC_CLI_DECODE_ONLY="1")


def test_cohort_decode_summaries_equal_single_runs(cohort):
    exe = _cli()
    s = cohort["samples"]
    inputs = [s["syn5a"], s["syn2"], s["test"], s["syn0"], s["syn5b"]]
    got, _ = _check_cohort_equals_single_runs(exe, cohort["dir"], "dec_l", ["-l", cohort["sites"]], inputs, [], DECODE_ONLY)
    assert all(o.count(b"\n") > 20 for o, _ in got[:2])
    # a site-list contig missing from one sample is reported in that sample's ERR only
    assert [b"chrC not found in bam file" in e for _, e in got] == [False, True, True, False, False]
    assert all(b"chrZ not found in bam file" in e and b"not found" not in o for o, e in got)
    # argv regions, parsed against each sample's own header; one long region cut into windows
    env = dict(DECODE_ONLY, BRC_CLI_WINDOW="5000")
    _check_cohort_equals_single_runs(exe, cohort["dir"], "dec_argv", [], inputs[:2] + inputs[3:], ["chrA:100-900", "chrA:500-23000", "chrA"], env)


def test_cohort_refuses_bad_lists_before_any_sample(cohort, tmp_path):
    exe = _cli()
    test = cohort["samples"]["test"]
    o1, o2 = str(tmp_path / "a.out"), str(tmp_path / "b.out")
    bad = {
        "one field": f"{test}\n",
        "four fields": f"{test}\t{o1}\t{o1}.e\textra\n",
        "empty field": f"{test}\t\t{o1}\n",
        "same OUT twice": f"{test}\t{o1}\n{test}\t{o1}\n",
        "OUT is an earlier ERR": f"{test}\t{o2}\t{o1}\n{test}\t{o1}\n",
        "OUT.log is an earlier OUT": f"{test}\t{o1}.log\n{test}\t{o1}\n",
        "OUT equals its ERR": f"{test}\t{o1}\t{o1}\n",
    }
    for why, text in bad.items():
        lst = tmp_path / "list"
        lst.write_text(f"{test}\t{tmp_path}/first.out\n" + text)
        p = subprocess.run([exe, "--bam-list", str(lst), "21:10402985-10402990"], capture_output=True, env=DECODE_ONLY)
        assert p.returncode == 1 and p.stderr, why
        assert not os.path.exists(tmp_path / "first.out"), why       # refused before the first sample ran
    lst.write_text(f"{test}\t{o1}\n")
    p = subprocess.run([exe, "--shard", "0/2", "--bam-list", str(lst), "21:10402985-10402990"], capture_output=True, env=DECODE_ONLY)
    assert p.returncode == 1 and b"--shard" in p.stderr and not os.path.exists(o1)
    p = subprocess.run([exe, "--bam-list", str(tmp_path / "no_such_list"), "21"], capture_output=True, env=DECODE_ONLY)
    assert p.returncode == 1 and b"no_such_list" in p.stderr


def test_cohort_failed_samples_do_not_stop_the_batch(cohort, tmp_path):
    exe = _cli()
    s = cohort["samples"]
    noidx = str(tmp_path / "noidx.bam")
    shutil.copy(s["test"], noidx)
    inputs = [str(tmp_path / "missing.bam"), noidx, s["cut"], s["syn2"], s["test"]]
    regions = ["21:10402000-10406000"]
    got, want = _check_cohort_equals_single_runs(exe, str(tmp_path), "fail", [], inputs, regions, DECODE_ONLY)
    assert [w[0] for w in want] == [1, 1, 1, 1, 0]
    assert b"Fail to open BAM file" in got[0][1] and b"BAM indexing file is not available." in got[1][1]
    assert b"truncated or corrupt" in got[2][1] and b"Invalid region 21:10402000-10406000" in got[3][1]
    assert got[4][0].count(b"\n") == 1 and got[4][1].startswith(b"Minimum mapping quality is set to 0\n")
    # ERR defaults to OUT.log
    rc, _, got2 = _run_cohort(exe, str(tmp_path), "deflog", [], [s["test"], s["test"]], regions, DECODE_ONLY, err_col=False)
    assert rc == 0 and got2[0] == got2[1] == got[4]


def test_cohort_cram_messages_of_htslib_go_to_the_sample_err(cohort, tmp_path):
    """htslib prints its own lines on stderr while it opens a CRAM and its index.  In a cohort they must land in that sample's
    ERR, in the same place among the host's lines as in the sample's own run; BAM samples opened ahead of their turn around
    them keep their ERR clean of them."""
    exe = _cli()
    if not _have_htslib(exe):
        pytest.skip("host built without htslib, or no CRAM fixture")
    s = cohort["samples"]
    cram = os.path.join(CRAM_DATA, "twolib.sorted.cram")
    inputs = [s["syn2"], s["cram_noidx"], s["test"], cram, str(tmp_path / "missing.cram"), s["cram_old_idx"], s["syn0"]]
    got, want = _check_cohort_equals_single_runs(exe, str(tmp_path), "cram", ["-f", cohort["fasta"], "-l", cohort["sites"]], inputs, [], DECODE_ONLY)
    assert [w[0] for w in want] == [0, 1, 0, 0, 1, 0, 0]
    assert b"Could not retrieve index file" in got[1][1] and b"Failed to open file" in got[4][1]
    for k in (0, 2, 3, 5, 6):
        assert b"[E::" not in got[k][1]


def test_cohort_outputs_are_opened_together(cohort, tmp_path):
    """A sample whose OUT or ERR cannot be opened fails alone and leaves no new file behind and no earlier file emptied."""
    exe = _cli()
    test = cohort["samples"]["test"]
    keep = tmp_path / "keep.out"
    keep.write_bytes(b"earlier output\n")
    lst = tmp_path / "list"
    lst.write_text(f"{test}\t{keep}\t{tmp_path}/no_dir/x.err\n{test}\t{tmp_path}/no_dir/y.out\t{tmp_path}/y.err\n{test}\t{tmp_path}/z.out\n")
    p = subprocess.run([exe, "--bam-list", str(lst), "21:10402985-10402990"], capture_output=True, env=DECODE_ONLY)
    assert p.returncode == 1 and p.stderr.count(b" failed: cannot open ") == 2, p.stderr
    assert keep.read_bytes() == b"earlier output\n" and not os.path.exists(tmp_path / "y.err")
    alone = subprocess.run([exe, test, "21:10402985-10402990"], capture_output=True, env=DECODE_ONLY)
    assert (tmp_path / "z.out").read_bytes() == alone.stdout and (tmp_path / "z.out.log").read_bytes() == alone.stderr


def test_cohort_window_jobs_pass_from_sample_to_sample(tmp_path):
    """Long regions are decoded by the parallel window path into the process's two window jobs, which every sample reuses;
    a sample after one that used them decodes its own first window at its turn.  Record summaries equal the single runs."""
    from bam_readcount_b200 import synth_cb
    exe = _cli()
    bams = []
    for k, seed in enumerate((5, 6)):
        d = tmp_path / f"s{k}"
        d.mkdir()
        bams.append(synth_cb.write_sample_bam(synth_cb.Spec(seed=seed, contig_len=1280 * 320), 0, 0, 320, str(d), _samtools())["bam"])
    env = dict(DECODE_ONLY, BRC_CLI_WINDOW="300000")
    regions = ["chr1:1-400000", "chr1:1001-2000"]
    got, _ = _check_cohort_equals_single_runs(exe, str(tmp_path), "win", [], [bams[0], bams[1], bams[0]], regions, env)
    assert got[0] == got[2] and got[0][0].count(b"\n") == 3
    rc, _, timed = _run_cohort(exe, str(tmp_path), "wint", [], [bams[0], bams[1], bams[0]], regions, dict(env, BRC_CLI_TIMING="1"))
    assert rc == 0 and all(b"windows decoded by" in e and b"(+ 0 records in 0 windows" not in e for _, e in timed)


def test_cohort_without_a_device_stops_at_the_first_sample(cohort, tmp_path):
    """No engine can be created: the first sample's ERR says why, as its single run does, and no later sample runs."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    exe = _cli()
    test = cohort["samples"]["test"]
    lst = tmp_path / "list"
    lst.write_text(f"{test}\t{tmp_path}/a.out\n{test}\t{tmp_path}/b.out\n")
    p = subprocess.run([exe, "-f", cohort["fasta"], "--bam-list", str(lst), "21:10402985-10402990"], capture_output=True)
    alone = subprocess.run([exe, "-f", cohort["fasta"], test, "21:10402985-10402990"], capture_output=True)
    assert p.returncode == alone.returncode == 1 and b"brc_create" in alone.stderr
    assert (tmp_path / "a.out.log").read_bytes() == alone.stderr and (tmp_path / "a.out").read_bytes() == alone.stdout
    assert not os.path.exists(tmp_path / "b.out") and b"not run" in p.stderr


# ---------------------------------------------------------------------------------------------------------------- GPU
FLAG_SETS = {
    "default": [], "p": ["-p"], "i": ["-i"], "ip": ["-i", "-p"], "q20b20": ["-q", "20", "-b", "20"], "d3": ["-d", "3"],
    "w2": ["-w", "2"], "alt2": ["--min-alt-count", "2"],
}


def _gpu_inputs(cohort, exe):
    """The cohort in an order that switches library counts (5, 2, 5, 0 ...) and @SQ orders from one sample to the next."""
    s = cohort["samples"]
    inputs = [s["syn5a"], s["syn2"], s["syn5b"], s["test"], s["syn0"], s["bad_rg"], s["cut"]]
    if _have_htslib(exe):
        inputs.insert(4, os.path.join(CRAM_DATA, "twolib.sorted.cram"))
        inputs.append(s["cram_noidx"])
    return inputs


@pytest.mark.gpu
@pytest.mark.parametrize("flags", list(FLAG_SETS))
def test_cohort_site_list_equals_single_runs(cohort, flags):
    exe = _cli()
    args = FLAG_SETS[flags] + ["-f", cohort["fasta"], "-l", cohort["sites"]]
    inputs = _gpu_inputs(cohort, exe)
    got, want = _check_cohort_equals_single_runs(exe, cohort["dir"], f"l_{flags}", args, inputs, [], dict(os.environ))
    assert [w[0] for w in want].count(1) == (2 if _have_htslib(exe) else 1)     # only the cut BAM and the CRAM without index fail
    golden = {"default": "expected_all_lib", "p": "expected_per_lib", "i": "expected_insertion_centric_all_lib",
              "ip": "expected_insertion_centric_per_lib", "w2": "expected_all_lib"}.get(flags)
    if golden:
        assert got[3][0].decode("latin-1") == cases.load_golden_text(golden)
    if flags == "w2":                                           # the -w cap is counted per sample
        for o, e in got[:1] + got[3:4]:
            assert e.count(b"has been emitted 2 times and will be disabled") >= 1


@pytest.mark.gpu
@pytest.mark.parametrize("flags", ["default", "p", "ip", "w2", "alt2"])
def test_cohort_argv_regions_equal_single_runs(cohort, flags):
    """Overlapping argv regions (the deletion queue is carried from one to the next inside a sample), and one long region
    cut into windows.  test.bam and the CRAM have no chrA: their runs fail on the region, in the cohort as alone."""
    exe = _cli()
    args = FLAG_SETS[flags] + ["-f", cohort["fasta"]]
    inputs = _gpu_inputs(cohort, exe)
    _check_cohort_equals_single_runs(exe, cohort["dir"], f"a_{flags}", args, inputs, ["chrA:1000-1300", "chrA:1200-1600", "chrA:1601-1700"], dict(os.environ))
    if flags in ("default", "p"):
        env = dict(os.environ, BRC_CLI_WINDOW="3777")
        got, _ = _check_cohort_equals_single_runs(exe, cohort["dir"], f"w_{flags}", args, inputs, ["chrA:1-24000"], env)
        assert got[0][0].count(b"\n") > 23000


@pytest.mark.gpu
def test_cohort_argv_regions_reproduce_reference_goldens(cohort):
    exe = _cli()
    s = cohort["samples"]
    regions = ["21:10402985-10402985", "21:10405200-10405200"]
    rc, _, got = _run_cohort(exe, cohort["dir"], "gold", ["-w", "1", "-f", cohort["fasta"]], [s["test"], s["bad_rg"], s["test"]], regions, dict(os.environ))
    assert rc == 0
    for o, _ in got:
        assert o.decode("latin-1") == cases.load_golden_text("expected_all_lib")


@pytest.mark.gpu
@pytest.mark.parametrize("flags", ["default", "p", "ip", "q20b20", "alt2"])
def test_cohort_device_decode_equals_single_runs(cohort, flags):
    exe = _cli()
    args = FLAG_SETS[flags] + ["-f", cohort["fasta"], "-l", cohort["sites"]]
    _check_cohort_equals_single_runs(exe, cohort["dir"], f"dev_{flags}", args, _gpu_inputs(cohort, exe), [], dict(os.environ, BRC_CLI_DEVICE_DECODE="1"))


@pytest.mark.gpu
def test_cohort_deletion_queue_does_not_cross_samples(tmp_path):
    """Sample A's deletion is anchored at the last site of its last argv region, so it sits in the carried queue when A ends.
    Sample B's first region starts at the next position: B's output must not show it."""
    exe = _cli()
    from bam_readcount_b200 import synth
    d = str(tmp_path)
    ref = synth.synth_reference(3000, 5)
    _write_fasta(os.path.join(d, "ref.fa"), [("chrA", ref.tobytes())])
    seq = lambda p, n: ref[p:p + n].tobytes().decode()               # noqa: E731
    def sam(name, reads):
        with open(os.path.join(d, name + ".sam"), "w") as fh:
            fh.write("@HD\tVN:1.6\tSO:coordinate\n@SQ\tSN:chrA\tLN:3000\n")
            for k, (pos, cigar, s) in enumerate(sorted(reads)):
                fh.write(f"r{k}\t0\tchrA\t{pos + 1}\t60\t{cigar}\t*\t0\t0\t{s}\t{'I' * len(s)}\tNM:i:0\n")
        bam = os.path.join(d, name + ".bam")
        subprocess.check_call([_samtools(), "view", "-b", "-o", bam, os.path.join(d, name + ".sam")])
        subprocess.check_call([_samtools(), "index", bam])
        return bam
    # A: 1-based 1001-1050 matched, 1051-1055 deleted, then 50 more; plus plain reads across the same stretch
    a = sam("a", [(1000, "50M5D50M", seq(1000, 50) + seq(1055, 50))] + [(980 + 7 * k, "100M", seq(980 + 7 * k, 100)) for k in range(6)])
    b = sam("b", [(990 + 5 * k, "100M", seq(990 + 5 * k, 100)) for k in range(8)])
    regions = ["chrA:1051-1060", "chrA:1000-1050"]
    got, want = _check_cohort_equals_single_runs(exe, d, "queue", ["-f", os.path.join(d, "ref.fa")], [a, b, a, b], regions, dict(os.environ))
    assert b"\t-" in got[0][0]                                  # A prints its own deletion (first region, from its halo site)
    assert b"\t-" not in got[1][0] and b"\t-" not in got[3][0]
    assert got[1][0].startswith(b"chrA\t1051\t")
