"""`brc-readcount --vcf FILE --vcf-samples LIST`: several sample columns of one VCF, each from its own input, in one process.
Sample NAME's column must hold exactly what `--vcf FILE --vcf-sample NAME INPUT` writes there, and its ERR (or, without one,
the process's STDERR) that run's STDERR.  CPU tests use the decode-only hook (BRC_CLI_DECODE_ONLY: per-region record
summaries on STDOUT and no VCF); GPU tests compare the VCF with the fold of the single-sample runs."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import cases
import vcf_cases
from cases import CONTIGS, CRAM_DATA, DECODE_ONLY, synthetic_bam

CRAM = os.path.join(CRAM_DATA, "twolib.sorted.cram")


def _records(seqs):
    """The --vcf fixture's records on 21 (and chrZ, a contig no input has), then SNVs, insertions and deletions at seeded
    positions of chrA/chrB/chrC and at the CRAM fixture's sites of rand1k."""
    recs = vcf_cases.fixture_records()
    rng = np.random.default_rng(5)
    for c, (L, _) in CONTIGS.items():
        for p in np.sort(rng.choice(np.arange(300, L - 300), 30, replace=False)):
            recs += _site_records(c, int(p), seqs[c])
    for p in range(45, 75, 3):
        recs += _site_records("rand1k", p, seqs["rand1k"])
    return recs


def _site_records(c, p, seq):
    r = seq[p - 1]
    return [(c, p, r, ",".join(b for b in "ACGT" if b != r)), (c, p, r, r + "A," + r + "TG"), (c, p, seq[p - 1:p + 1], r),
            (c, p, seq[p - 1:p + 2], r)]


@pytest.fixture(scope="module")
def cohort(tmp_path_factory):
    """Synthetic BAMs with 5, 2 and 0 libraries, different @SQ orders and contig subsets; the reference's test.bam; test.bam cut
    inside a BGZF block; test.bam without its index; one FASTA holding every contig; the records of every contig."""
    from bam_readcount_b200 import synth
    d = str(tmp_path_factory.mktemp("vcf_samples"))
    s = {
        "syn5": synthetic_bam(d, "syn5", ["chrA", "chrB", "chrC"], 5, seed=21, no_nm=60),
        "syn2": synthetic_bam(d, "syn2", ["chrB", "chrA"], 2, seed=22),
        "syn0": synthetic_bam(d, "syn0", ["chrA", "chrC"], 0, seed=24, no_nm=10),
        "test": os.path.join(cases.GOLDEN, "test.bam"),
    }
    s["cut"] = os.path.join(d, "cut.bam")
    with open(s["test"], "rb") as fh:
        open(s["cut"], "wb").write(fh.read()[:60000])
    shutil.copy(s["test"] + ".bai", s["cut"] + ".bai")
    s["noidx"] = os.path.join(d, "noidx.bam")
    shutil.copy(s["test"], s["noidx"])
    rand1k = b"".join(open(os.path.join(cases.GOLDEN, "rand1k.fa"), "rb").read().split(b"\n")[1:])
    seqs = {"21": cases.testbam_chr21(), "rand1k": rand1k}
    seqs.update({c: synth.synth_reference(L, sd).tobytes() for c, (L, sd) in CONTIGS.items()})
    fa = cases.write_fasta(os.path.join(d, "all.fa"), list(seqs.items()))
    recs = _records({c: v.decode("latin-1").upper() for c, v in seqs.items()})
    return dict(dir=d, samples=s, fasta=fa, records=recs)


def _write_vcf(d, tag, cohort, columns, bgzf=False):
    """The records as a VCF with sample columns `columns` (None: sites-only); its path and text."""
    text = vcf_cases.vcf_text(cohort["records"], samples=columns or ("S1",), sites_only=columns is None)
    path = os.path.join(d, f"{tag}.vcf" + (".gz" if bgzf else ""))
    if bgzf:
        vcf_cases.write_bgzf(path, text.encode())
    else:
        open(path, "w").write(text)
    return path, text


def _run_list(exe, d, tag, args, vcf, samples, env, err_col=True):
    """One --vcf-samples run over `samples` [(NAME, INPUT)]; returns (exit status, STDOUT, STDERR, [ERR bytes or None])."""
    lst = os.path.join(d, f"{tag}.list")
    errs = [os.path.join(d, f"{tag}.{k}.err") if err_col else None for k in range(len(samples))]
    with open(lst, "w") as fh:
        for k, (name, inp) in enumerate(samples):
            fh.write(f"{name}\t{inp}" + (f"\t{errs[k]}" if err_col else "") + ("\r\n" if k == 0 else "\n"))
            if k == 1:
                fh.write("\n")                                  # empty lines are skipped
    p = subprocess.run([exe] + args + ["--vcf", vcf, "--vcf-samples", lst], capture_output=True, env=env)
    return p.returncode, p.stdout, p.stderr, [open(e, "rb").read() if e and os.path.exists(e) else None for e in errs]


def _single(exe, args, vcf, name, inp, env):
    p = subprocess.run([exe] + args + ["--vcf", vcf, "--vcf-sample", name, inp], capture_output=True, env=env)
    return p.returncode, p.stdout, p.stderr


def _singles(exe, args, vcf, samples, env):
    return [_single(exe, args, vcf, name, inp, env) for name, inp in samples]


def _fold(text, names, outs):
    """The VCF the single-sample runs imply: header lines and columns 0-8 from the single runs, each listed column from its
    own run, unlisted columns from the input; a sites-only VCF gets a FORMAT column and one column per name in list order."""
    runs = [o.decode("latin-1").splitlines() for o in outs]
    hc = [ln for ln in text.splitlines() if ln.startswith("#CHROM")][0].split("\t")
    body = [ln.split("\t") for ln in text.splitlines() if not ln.startswith("#")]
    sites_only = len(hc) == 8
    out, k = [], 0
    for i, ln in enumerate(runs[0]):
        assert all(len(r) == len(runs[0]) for r in runs)
        if ln.startswith("##"):
            assert all(r[i] == ln for r in runs)
            out.append(ln)
        elif ln.startswith("#CHROM"):
            out.append("\t".join(hc + (["FORMAT"] + list(names) if sites_only else [])))
        else:
            mine = ln.split("\t")
            cols = mine[:9] if sites_only else mine[:9] + body[k][9:]
            for n, r in zip(names, runs):
                v = r[i].split("\t")[9 if sites_only else hc.index(n)]
                if sites_only:
                    cols.append(v)
                else:
                    cols[hc.index(n)] = v
            out.append("\t".join(cols))
            k += 1
    assert k == len(body)
    return ("\n".join(out) + "\n").encode("latin-1")


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_refusals_before_any_sample(cohort, tmp_path):
    """Each refusal exits 1 with a message, prints nothing on STDOUT, creates no ERR and leaves an existing ERR as it was."""
    exe = cases.cli()
    s = cohort["samples"]
    vcf, _ = _write_vcf(str(tmp_path), "two", cohort, ("S1", "S2"))
    dup, _ = _write_vcf(str(tmp_path), "dup", cohort, ("S1", "S2", "S1"))
    keep, new = tmp_path / "keep.err", tmp_path / "new.err"
    keep.write_bytes(b"earlier\n")
    good = f"S1\t{s['test']}\t{keep}\nS2\t{s['syn2']}\t{new}\n"
    lists = {
        "one field": (good + "S3\n", b"a sample line is NAME<TAB>INPUT"),
        "four fields": (good + f"S3\t{s['test']}\t{tmp_path}/x.err\textra\n", b"a sample line is NAME<TAB>INPUT"),
        "empty field": (good + f"S3\t\t{tmp_path}/x.err\n", b"a sample line is NAME<TAB>INPUT"),
        "empty list": ("\n\n", b"lists no sample"),
        "name twice": (good + f"S1\t{s['syn0']}\n", b"sample S1 is listed twice"),
        "err twice": (good + f"S3\t{s['syn0']}\t{tmp_path}/sub/../keep.err\n", b"is already the output of an earlier sample"),
        "no such column": (good + f"S9\t{s['syn0']}\n", b"--vcf-samples S9: no such sample"),
    }
    lst = tmp_path / "list"

    def refused(args, msg, why):
        p = subprocess.run([exe] + args, capture_output=True, env=DECODE_ONLY)
        assert p.returncode == 1 and msg in p.stderr and p.stdout == b"", (why, p.stderr)
        assert keep.read_bytes() == b"earlier\n" and not new.exists(), why

    for why, (text, msg) in lists.items():
        lst.write_text(text)
        refused(["--vcf", vcf, "--vcf-samples", str(lst)], msg, why)
    lst.write_text(good)
    refused(["--vcf", dup, "--vcf-samples", str(lst)], b"--vcf-samples S1 is ambiguous: 2 sample columns", "ambiguous")
    refused(["--vcf", vcf, "--vcf-samples", str(tmp_path / "no_such_list")], b"Failed to open sample list file", "unreadable")
    refused(["--vcf-samples", str(lst)], b"--vcf-samples needs --vcf", "no --vcf")
    refused(["--vcf", vcf, "--vcf-sample", "S1", "--vcf-samples", str(lst)], b"cannot be combined with --vcf-sample", "--vcf-sample")
    refused(["--vcf", vcf, "--vcf-samples", str(lst), s["test"]], b"takes no positional argument", "positional")
    refused(["--vcf", vcf, "--vcf-samples", str(lst), "21:1-100"], b"takes no positional argument", "region")
    for extra, what in ((["-l", vcf], b"-l"), (["-p"], b"-p"), (["--min-alt-count", "2"], b"--min-alt-count"),
                        (["--min-alt-fraction", "0.1"], b"--min-alt-count/--min-alt-fraction"), (["--shard", "0/2"], b"--shard"),
                        (["--bam-list", str(lst)], b"--bam-list")):
        refused(extra + ["--vcf", vcf, "--vcf-samples", str(lst)], b"--vcf cannot be combined with " + what, extra)


@pytest.mark.parametrize("columns", [("S1", "S2", "S3", "S4", "S5"), None])
def test_decode_summaries_equal_single_runs(cohort, tmp_path, columns):
    """Each sample derives its site list against its own header: STDOUT is the single runs' decode summaries in list order, and
    each ERR is that run's STDERR, with the 'not found in bam file' lines of the contigs that input lacks."""
    exe = cases.cli()
    s = cohort["samples"]
    vcf, _ = _write_vcf(str(tmp_path), "in", cohort, columns)
    names = ["S4", "S1", "S5", "S3"] if columns else ["T", "N", "X", "Y"]
    samples = list(zip(names, [s["syn5"], s["syn2"], s["test"], s["syn0"]]))
    args = ["-f", cohort["fasta"]]
    want = _singles(exe, args, vcf, samples, DECODE_ONLY)
    rc, out, err, errs = _run_list(exe, str(tmp_path), "dec", args, vcf, samples, DECODE_ONLY)
    assert rc == 0 and [w[0] for w in want] == [0] * 4, err.decode()
    assert out == b"".join(w[1] for w in want) and out.count(b"\n") > 100
    assert errs == [w[2] for w in want] and err == b""
    assert [b"chrC not found in bam file" in e for e in errs] == [False, True, True, False]
    assert [b"21 not found in bam file" in e for e in errs] == [True, True, False, True]
    assert all(b"chrZ not found in bam file" in e for e in errs)
    # without ERR files the process's STDERR is the single runs' STDERRs in list order
    rc, out2, err2, _ = _run_list(exe, str(tmp_path), "dec_noerr", args, vcf, samples, DECODE_ONLY, err_col=False)
    assert rc == 0 and out2 == out and err2 == b"".join(w[2] for w in want)
    # the same input under two names: the same summary twice
    rc, out3, _, errs3 = _run_list(exe, str(tmp_path), "dec_twice", args, vcf, [samples[1], (samples[0][0], samples[1][1])], DECODE_ONLY)
    assert rc == 0 and out3 == want[1][1] * 2 and errs3 == [want[1][2]] * 2


@pytest.mark.parametrize("bad", ["cut", "noidx"])
def test_failed_sample_does_not_stop_the_others(cohort, tmp_path, bad):
    exe = cases.cli()
    s = cohort["samples"]
    vcf, _ = _write_vcf(str(tmp_path), "in", cohort, ("S1", "S2", "S3"))
    samples = [("S2", s["syn5"]), ("S1", s[bad]), ("S3", s["test"])]
    args = ["-f", cohort["fasta"]]
    want = _singles(exe, args, vcf, samples, DECODE_ONLY)
    assert [w[0] for w in want] == [0, 1, 0]
    rc, out, err, errs = _run_list(exe, str(tmp_path), "fail", args, vcf, samples, DECODE_ONLY)
    assert rc == 1 and out == b"".join(w[1] for w in want) and errs == [w[2] for w in want]
    assert err.decode().splitlines() == [f"sample 2 ({s[bad]}) failed: see {tmp_path}/fail.1.err"]
    assert (b"truncated or corrupt" if bad == "cut" else b"BAM indexing file is not available.") in errs[1]
    # without ERR files: the failure line follows the failed sample's own lines
    rc, out, err, _ = _run_list(exe, str(tmp_path), "fail_noerr", args, vcf, samples, DECODE_ONLY, err_col=False)
    assert rc == 1 and out == b"".join(w[1] for w in want)
    assert err == want[0][2] + want[1][2] + f"sample 2 ({s[bad]}) failed: see the lines above\n".encode() + want[2][2]


def test_unwritable_err_fails_that_sample_alone(cohort, tmp_path):
    exe = cases.cli()
    s = cohort["samples"]
    vcf, _ = _write_vcf(str(tmp_path), "in", cohort, ("S1", "S2"))
    lst = tmp_path / "list"
    lst.write_text(f"S1\t{s['syn2']}\t{tmp_path}/no_dir/a.err\nS2\t{s['test']}\t{tmp_path}/b.err\n")
    p = subprocess.run([exe, "--vcf", vcf, "--vcf-samples", str(lst)], capture_output=True, env=DECODE_ONLY)
    want = _single(exe, [], vcf, "S2", s["test"], DECODE_ONLY)
    assert p.returncode == 1 and p.stderr.count(b" failed: cannot open ") == 1, p.stderr
    assert p.stdout == want[1] and (tmp_path / "b.err").read_bytes() == want[2]


def test_without_a_device_stops_at_the_first_sample(cohort, tmp_path):
    """No engine can be created: the first sample's ERR says why, as its single run does, no later sample runs and no VCF is
    written."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    exe = cases.cli()
    s = cohort["samples"]
    vcf, _ = _write_vcf(str(tmp_path), "in", cohort, ("S1", "S2"))
    args = ["-f", cohort["fasta"]]
    rc, out, err, errs = _run_list(exe, str(tmp_path), "nodev", args, vcf, [("S1", s["test"]), ("S2", s["syn2"])], dict(os.environ))
    alone = _single(exe, args, vcf, "S1", s["test"], dict(os.environ))
    assert rc == alone[0] == 1 and b"brc_create" in alone[2] and out == b"" == alone[1]
    assert errs[0] == alone[2] and errs[1] is None and b"not run" in err


# ---------------------------------------------------------------------------------------------------------------- GPU
FLAG_SETS = {"default": [], "i": ["-i"], "q20b20": ["-q", "20", "-b", "20"], "w2": ["-w", "2"]}


def _check_fold(exe, cohort, d, tag, args, vcf, text, samples, env):
    """One --vcf-samples run against the single-sample runs: STDOUT is their fold, each ERR is its run's STDERR."""
    want = _singles(exe, args, vcf, samples, env)
    assert [w[0] for w in want] == [0] * len(samples), [w[2].decode()[-500:] for w in want]
    rc, out, err, errs = _run_list(exe, d, tag, args, vcf, samples, env)
    assert rc == 0, err.decode()
    assert out == _fold(text, [n for n, _ in samples], [w[1] for w in want])
    assert errs == [w[2] for w in want]
    return out, want


@pytest.mark.gpu
@pytest.mark.parametrize("flags", list(FLAG_SETS))
@pytest.mark.parametrize("shape", ["two", "three_one_unlisted", "sites_only", "bgzf", "device_decode"])
def test_vcf_samples_fold_of_single_runs(cohort, tmp_path, flags, shape):
    exe = cases.cli()
    s = cohort["samples"]
    columns, samples = {
        "two": (("S1", "S2"), [("S1", s["syn5"]), ("S2", s["test"])]),
        "three_one_unlisted": (("S1", "S2", "S3"), [("S3", s["syn2"]), ("S1", s["syn0"])]),
        "sites_only": (None, [("N1", s["test"]), ("N2", s["syn5"]), ("N3", s["syn2"])]),
        "bgzf": (("S1", "S2"), [("S1", s["syn2"]), ("S2", s["test"])]),
        "device_decode": (("S1", "S2"), [("S1", s["syn5"]), ("S2", s["syn0"])]),
    }[shape]
    vcf, text = _write_vcf(str(tmp_path), "in", cohort, columns, bgzf=shape == "bgzf")
    env = dict(os.environ, BRC_CLI_DEVICE_DECODE="1") if shape == "device_decode" else dict(os.environ)
    out, want = _check_fold(exe, cohort, str(tmp_path), shape, FLAG_SETS[flags] + ["-f", cohort["fasta"]], vcf, text, samples, env)
    # every listed column has records with reads (a DP above 0)
    rows = [ln.split("\t") for ln in out.decode().splitlines() if not ln.startswith("#")]
    cols = [9 + k for k in range(len(samples))] if columns is None else [columns.index(n) + 9 for n, _ in samples]
    for c in cols:
        assert any(r[c].split(":")[-5] not in (".", "0") for r in rows), (shape, c)
    if flags == "w2" and samples[0][1] == s["syn5"] and shape != "device_decode":
        assert b"has been emitted 2 times and will be disabled" in want[0][2]


@pytest.mark.gpu
def test_vcf_samples_one_input_under_two_names(cohort, tmp_path):
    exe = cases.cli()
    s = cohort["samples"]
    vcf, text = _write_vcf(str(tmp_path), "in", cohort, ("S1", "S2", "S3"))
    out, _ = _check_fold(exe, cohort, str(tmp_path), "twice", ["-f", cohort["fasta"]], vcf, text, [("S1", s["syn5"]), ("S3", s["syn5"])], dict(os.environ))
    rows = [ln.split("\t") for ln in out.decode().splitlines() if not ln.startswith("#")]
    assert all(r[9] == r[11] for r in rows) and any(r[9].split(":")[2] not in (".", "0") for r in rows)


@pytest.mark.gpu
@pytest.mark.parametrize("flags", ["default", "w2"])
def test_vcf_samples_list_order_does_not_matter(cohort, tmp_path, flags):
    """Reversed, the list gives the same VCF and the same ERRs: no deletion queue, reference window or warning state passes from
    one sample to the next."""
    exe = cases.cli()
    s = cohort["samples"]
    vcf, _ = _write_vcf(str(tmp_path), "in", cohort, ("S1", "S2", "S3", "S4"))
    samples = [("S1", s["syn5"]), ("S2", s["test"]), ("S3", s["syn2"]), ("S4", s["syn0"])]
    args = FLAG_SETS[flags] + ["-f", cohort["fasta"]]
    rc, out, err, errs = _run_list(exe, str(tmp_path), "fwd", args, vcf, samples, dict(os.environ))
    rc2, out2, err2, errs2 = _run_list(exe, str(tmp_path), "rev", args, vcf, samples[::-1], dict(os.environ))
    assert rc == rc2 == 0, (err + err2).decode()
    assert out == out2 and errs == errs2[::-1]


@pytest.mark.gpu
def test_vcf_samples_failed_sample_between_good_ones(cohort, tmp_path):
    exe = cases.cli()
    s = cohort["samples"]
    vcf, text = _write_vcf(str(tmp_path), "in", cohort, ("S1", "S2", "S3"))
    args = ["-f", cohort["fasta"]]
    samples = [("S1", s["syn5"]), ("S2", s["cut"]), ("S3", s["test"])]
    want = _singles(exe, args, vcf, samples, dict(os.environ))
    assert [w[0] for w in want] == [0, 1, 0]
    rc, out, err, errs = _run_list(exe, str(tmp_path), "fail", args, vcf, samples, dict(os.environ))
    assert rc == 1 and err.count(b" failed") == 1 and errs == [w[2] for w in want]
    # the failed sample's column: its existing keys padded to FORMAT's, then '.' in all five fields
    good = _fold(text, ["S1", "S3"], [want[0][1], want[2][1]]).decode().splitlines()
    got = out.decode().splitlines()
    assert len(got) == len(good)
    for g, w in zip(got, good):
        if g.startswith("#"):
            assert g == w
            continue
        gc, wc = g.split("\t"), w.split("\t")
        assert gc[:10] + gc[11:] == wc[:10] + wc[11:]
        assert gc[10] == wc[10] + ":.:.:.:.:."                  # the input's GT:GQ, as the FORMAT keys need no padding


@pytest.mark.gpu
def test_vcf_samples_cram(cohort, tmp_path):
    if not (cases.have_htslib() and os.path.exists(CRAM)):
        pytest.skip("host built without htslib, or no CRAM fixture")
    exe = cases.cli()
    s = cohort["samples"]
    vcf, text = _write_vcf(str(tmp_path), "in", cohort, ("S1", "S2", "S3"))
    samples = [("S2", s["syn2"]), ("S1", CRAM), ("S3", s["test"])]
    out, want = _check_fold(exe, cohort, str(tmp_path), "cram", ["-f", cohort["fasta"]], vcf, text, samples, dict(os.environ))
    rows = [ln.split("\t") for ln in out.decode().splitlines() if ln.startswith("rand1k")]
    assert rows and any(r[9].split(":")[2] not in (".", "0") for r in rows)
