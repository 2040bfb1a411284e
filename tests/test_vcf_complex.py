"""GPU: complex-record queries (brc_set_complex_queries) and `brc-readcount --vcf --vcf-complex`.

Engine: the answers equal tests/complex_rule.py on the admitted reads of each record's line, under the default flags, -q 20
-b 20, -i and -d 5, on a crafted MNP, a 30x synthetic contig with thousands of records, a 50 000x site, the pipelined push path,
brc_run_device over a multi-Mb region; allele queries of the same batch answer as they do alone.  CLI: --vcf --vcf-complex is
complex_rule.annotate over the text of `-l <derived>`, every other record's line is plain --vcf's, STDERR is `-l derived`'s,
and each --vcf-samples column is its own single run's."""
import bisect
import os
import subprocess

import numpy as np
import pytest

import cases
import complex_cases
import complex_rule
import vcf_cases
from bam_readcount_b200.engine import CRegion

pytestmark = pytest.mark.gpu

FLAGS = {"default": {}, "q20b20": dict(min_mapq=20, min_bq=20), "ic": dict(insertion_centric=True), "d5": dict(max_cnt=5)}


def _queries(records):
    """Per record of the batch (region g = its index): complex queries, and allele queries for the per-site records."""
    cq, aq, keys = [], [], []
    for g, (chrom, pos, ref, alt) in enumerate(records):
        cx = complex_rule.complex_alleles(pos, ref, alt.split(","))
        if cx is None:
            if len(ref) == 1 and len(alt) == 1:        # an SNV: its REF and ALT entries
                aq += [(g, pos - 1, "=ACGTN".index(ref.upper()), 0), (g, pos - 1, "=ACGTN".index(alt.upper()), 0)]
            continue
        al = [cx[0]] + [a for a in cx[1] if a is not None]
        cq.append((g, pos - 1, len(cx[0]), al))
        keys.append((pos - 1, len(cx[0]), tuple(al)))
    return cq, aq, keys


def _check(e, cq, keys, want):
    depth, counts = e.complex_answers()
    assert len(depth) == len(cq) and len(counts) == sum(len(q[3]) for q in cq)
    a = 0
    for i, k in enumerate(keys):
        dp, cnt = want[k]
        n = len(k[2])
        got = [(int(c["count"]), int(c["plus"]), int(c["count"] - c["plus"])) for c in counts[a:a + n]]
        assert (int(depth[i]), got) == (dp, cnt), (k, int(depth[i]), got, dp, cnt)
        a += n


def _engine_check(case, records, flags, reads=None, push="one"):
    """One region per record; the allele answers alone, then with the complex queries of the same batch."""
    regions = [(0, pos, pos) for _, pos, _, _ in records]
    cq, aq, keys = _queries(records)
    want = complex_cases.rule_answers(case, records, flags, reads)
    with cases.open_engine(case, flags) as e:
        cases.push_regions(e, case, True, regions=regions, push=push)
        e.set_allele_queries(aq)
        assert e.compute() is None
        alone, launches = e.allele_answers(), e.launch_count()
        e.reset()
        cases.push_regions(e, case, True, regions=regions, push=push)
        e.set_complex_queries(cq)
        e.set_allele_queries(aq)
        assert e.compute() is None
        assert (e.allele_answers() == alone).all()
        _check(e, cq, keys, want)
        assert e.launch_count() == launches + 1 and e.stage_ms(5) > 0.0
    nz = sum(1 for k in keys if want[k][0] > 0 and any(c[0] for c in want[k][1][1:]))
    return len(keys), nz


@pytest.mark.parametrize("flags", list(FLAGS))
def test_crafted(tmp_path, flags):
    case = complex_cases.crafted_case(str(tmp_path))
    recs = complex_cases.crafted_records()
    n, nz = _engine_check(case, recs, dict(FLAGS[flags]))
    assert n == 4 and nz >= 2
    # the IUPAC read is counted for the allele that spells its R as N
    r = complex_cases.crafted_alleles()[0]
    want = complex_cases.rule_answers(case, recs, dict(FLAGS[flags]))
    key = [k for k in want if r[0] + "N" in k[2]][0]
    i = key[2].index(r[0] + "N")
    assert want[key][1][i][0] == (0 if flags == "d5" else 1)


_SYN = {}


def _synthetic():
    if not _SYN:
        case = cases.synthetic_case(L=265000, depth=30, seed=21, regions=[], n_libs=1)
        recs = complex_cases.synthetic_records(case, 13000, seed=21)
        _SYN.update(case=case, records=recs, reads=complex_rule.Reads(case["batch"]))
    return _SYN


@pytest.mark.parametrize("flags", list(FLAGS))
def test_synthetic_contig(flags):
    s = _synthetic()
    fl = dict(FLAGS[flags])
    recs = s["records"] if flags != "d5" else s["records"][:1500]     # -d: the rule takes each line's admitted reads
    n, nz = _engine_check(s["case"], recs, fl, reads=None if flags == "d5" else s["reads"])
    # under -b 20 a long span rarely has every base at quality 20: fewer ALTs are seen
    assert n >= (1000 if flags == "d5" else 10000) and nz > (n // 40 if flags == "q20b20" else n // 2)


@pytest.mark.parametrize("flags", ["default", "q20b20"])
def test_deep_site(flags):
    """One record at 50 000x: far past the 2 048-read threshold of the deep-site kernel, one warp walks every read."""
    case = cases.deep_case(n_sites=1, depth=50000, seed=22, n_libs=1)
    site = case["regions"][0][1] - 1
    ref = case["contigs"][0][2].decode()
    reads = complex_rule.Reads(case["batch"])
    alts = set()
    for row in reads.rows[:3000]:
        f = complex_rule.resolve(row[4], row[0], site - 1, site + 3)
        if f is not None and row[5][f[0] + 1:f[1]] != ref[site:site + 3]:
            alts.add(row[5][f[0] + 1:f[1]])
    recs = [("chr1", site + 1, ref[site:site + 3], ",".join(sorted(a for a in alts if complex_rule._acgtn(a))[:40] + ["TTTT"]))]
    n, nz = _engine_check(case, recs, dict(FLAGS[flags]), reads=reads)
    dp = complex_cases.rule_answers(case, recs, dict(FLAGS[flags]), reads)
    assert n == 1 and nz == 1 and list(dp.values())[0][0] >= (25000 if flags == "default" else 5000)


@pytest.mark.parametrize("flags", ["default", "q20b20"])
def test_pipelined_chunks(monkeypatch, flags):
    """One long borrowed region streamed through the GPU in 7 chunks (compute_pipelined), its queries spread over it."""
    monkeypatch.setenv("BRC_PIPE_CHUNKS", "7")
    case = cases.synthetic_case(L=30000, depth=30, seed=23, regions=[(0, 2000, 26000)], n_libs=1)
    recs = [r for r in complex_cases.synthetic_records(case, 1300, seed=23) if 2000 <= r[1] < 26000 and
            complex_rule.complex_alleles(r[1], r[2], r[3].split(","))]
    cq, _, keys = _queries(recs)
    cq = [(0, p, n, al) for _, p, n, al in cq]
    want = complex_cases.rule_answers(case, recs, FLAGS[flags], complex_rule.Reads(case["batch"]))
    with cases.open_engine(case, FLAGS[flags]) as e:
        cases.push_regions(e, case, False)
        e.set_complex_queries(cq)
        assert e.compute() is None
        _check(e, cq, keys, want)
    assert len(cq) > 900


@pytest.mark.parametrize("flags", ["default", "q20b20"])
def test_device_path(flags):
    """brc_plan_device / brc_run_device over a 2.5 Mb region leave the answers on the device; brc_fetch_device_results copies
    them."""
    import torch
    case = cases.synthetic_case(L=2_500_000, depth=8, seed=24, regions=[(0, 1000, 2_490_000)], n_libs=1)
    rng = np.random.default_rng(24)
    ref = case["contigs"][0][2].decode()
    tid, beg, end, sub, first_pos, n_slots, _ = cases.region_geometry(case, case["regions"][0])
    pos0 = np.sort(rng.choice(np.arange(2000, 2_480_000), 400, replace=False))
    near = np.unique(np.concatenate([np.nonzero(np.abs(sub.pos.astype(np.int64) - p) < 200)[0] for p in pos0]))
    reads = complex_rule.Reads(sub, near)
    recs = []
    for p in pos0.tolist():
        n = int(rng.integers(1, 8))
        alts = {row[5][f[0] + 1:f[1]] for row in reads.rows[bisect.bisect_left(reads.starts, p - 160):bisect.bisect_left(reads.starts, p)]
                for f in [complex_rule.resolve(row[4], row[0], p - 1, p + n)] if f is not None}
        alts = sorted(a for a in alts if complex_rule._acgtn(a) and a != ref[p:p + n])[:3] + ["".join(complex_cases._other(b) for b in ref[p:p + n]) + "C"]
        recs.append(("chr1", p + 1, ref[p:p + n], ",".join(alts)))
    cq, _, keys = _queries(recs)
    cq = [(0, p, n, al) for _, p, n, al in cq]
    want = complex_cases.rule_answers(case, recs, FLAGS[flags], reads)
    with cases.open_engine(case, FLAGS[flags]) as e:
        cb, keep = cases.device_batch(sub, torch.device("cuda:0"))
        stream = torch.cuda.Stream()
        e.plan_device([CRegion(tid, beg, end, 0, 0, sub.n_reads, 0, first_pos, n_slots)], sub.n_reads, 1 << 22)
        e.set_complex_queries(cq)
        e.run_device(cb, None, stream.cuda_stream)
        assert e.fetch_device_results(stream.cuda_stream) is None
        _check(e, cq, keys, want)
        assert e.stage_ms(5) > 0.0
    assert sum(1 for k in keys if want[k][0]) > (300 if flags == "default" else 150)


@pytest.mark.parametrize("flags", ["default", "q20b20", "ic"])
def test_device_decoded_span(flags):
    """brc_push_bam_span: each record's line fetched as a compressed span of test.bam and decoded on the device."""
    from bam_readcount_b200 import bamio
    bam = os.path.join(cases.GOLDEN, "test.bam")
    hdr, _ = bamio.read_bam(bam)
    rg_lib = {rg: hdr.lib_of_rg(rg) for rg in hdr.rg_lb}
    bai = bamio.BaiIndex(bam + ".bai")
    case = cases.testbam_case()
    recs = [r for r in vcf_cases.fixture_records() if r[0] == "21" and complex_rule.complex_alleles(r[1], r[2], r[3].split(","))]
    want = complex_cases.rule_answers(case, recs, FLAGS[flags])
    tid = cases.case_tid(case, 0)
    with cases.open_engine(case, FLAGS[flags]) as e:
        for rec in recs:
            cq, _, keys = _queries([rec])
            e.reset()
            e.begin_region(tid, rec[1] - 1, rec[1], True)
            e.push_bam_span(bamio.bam_span(bam, bai, tid, rec[1] - 2, rec[1], rg_lib))
            e.end_region()
            e.set_complex_queries(cq)
            assert e.compute() is None
            _check(e, cq, keys, want)
    assert len(recs) >= 20 and sum(1 for v in want.values() if v[0]) >= 10


def test_refusals_and_reset():
    import ctypes as C
    from bam_readcount_b200.engine import RESULTS_ANSWERS, RESULTS_DENSE, RESULTS_NONE, BrcError, CResults
    case = cases.synthetic_case(L=6000, depth=20, seed=25, regions=[(0, 500, 1500)], n_libs=2)   # prints sites [499, 1500)
    with cases.open_engine(case, dict(per_lib=True)) as e:
        cases.push_regions(e, case, True)
        with pytest.raises(BrcError):
            e.set_complex_queries([(0, 600, 2, ["AC"])])
    with cases.open_engine(case) as e:
        cases.push_regions(e, case, True)
        e.compute()
        plain_text, plain_launches = e.format_text(-1), e.launch_count()
    with cases.open_engine(case) as e:
        e.set_site_filter(1, 0.0)
        cases.push_regions(e, case, True)
        with pytest.raises(BrcError):
            e.set_complex_queries([(0, 600, 2, ["AC"])])
        e.clear_site_filter()
        for bad in ([(1, 600, 2, ["AC"])], [(0, 498, 2, ["AC"])], [(0, 1500, 2, ["AC"])], [(0, 600, 0, ["AC"])], [(0, 600, 2, [])],
                    [(0, 600, 2, ["AR"])], [(0, 600, 2, [""])]):
            with pytest.raises(BrcError):
                e.set_complex_queries(bad)
            assert e.results_kind() == RESULTS_NONE
        from bam_readcount_b200.engine import CComplexAllele, CComplexQuery
        qa = (CComplexQuery * 1)(CComplexQuery(0, 600, 2, 2, 0))
        aa = (CComplexAllele * 1)(CComplexAllele(0, 2, 0))
        assert e.lib.brc_set_complex_queries(e.h, qa, 1, aa, 1, b"AC", 2) != 0           # allele counts do not add up
        aa2 = (CComplexAllele * 1)(CComplexAllele(1, 2, 0))
        qa1 = (CComplexQuery * 1)(CComplexQuery(0, 600, 2, 1, 0))
        assert e.lib.brc_set_complex_queries(e.h, qa1, 1, aa2, 1, b"AC", 2) != 0         # bases outside the buffer
        e.set_complex_queries([(0, 600, 2, ["AC", "GT"])])
        with pytest.raises(BrcError):
            e.set_site_filter(1, 0.0)
        assert e.lib.brc_compute(e.h) == 0
        assert e.results_kind() == RESULTS_ANSWERS
        assert e.lib.brc_get_results(e.h, C.byref(CResults())) != 0
        d, c = e.complex_answers()
        assert len(d) == 1 and len(c) == 2 and len(e.allele_answers()) == 0 and e.stage_ms(5) > 0.0 and e.stage_ms(4) >= 0.0
        e.set_complex_queries([(0, 600, 2, ["AC"])])          # queries of a next run drop the answers of the last one
        assert e.results_kind() == RESULTS_NONE and e.stage_ms(5) == 0.0
        e.reset()
        assert e.results_kind() == RESULTS_NONE
        cases.push_regions(e, case, True)
        e.compute()
        assert e.results_kind() == RESULTS_DENSE
        assert e.format_text(-1) == plain_text and e.launch_count() == plain_launches and e.stage_ms(5) == 0.0


# ---------------------------------------------------------------------------------------------------------------- CLI
def _testbam_answers(text, flags):
    case = cases.testbam_case()
    recs = [tuple(ln.split("\t")[:2]) + tuple(ln.split("\t")[3:5]) for ln in text.splitlines() if ln and ln[0] != "#"]
    recs = [(c, int(p), r, a) for c, p, r, a in recs if c == "21"]
    want = complex_cases.rule_answers(case, recs, flags)
    return lambda chrom, pos0, n, al: want[(pos0, n, tuple(al))]


CLI_FLAGS = {"default": ([], {}), "ic": (["-i"], {}), "q20b20": (["-q", "20", "-b", "20"], dict(min_mapq=20, min_bq=20)),
             "d5": (["-d", "5"], dict(max_cnt=5))}


@pytest.mark.parametrize("flags", list(CLI_FLAGS))
@pytest.mark.parametrize("shape", ["one", "sites_only", "device_decode"])
def test_cli_fixture(tmp_path, flags, shape):
    if shape == "device_decode" and flags == "d5":
        pytest.skip("the device-decoded span path needs a -d above the region's read count")
    exe = cases.cli()
    fa = cases.write_testbam_fasta(str(tmp_path / "ref.fa"))
    bam = os.path.join(cases.GOLDEN, "test.bam")
    argv, fl = CLI_FLAGS[flags]
    text = vcf_cases.vcf_text(vcf_cases.fixture_records(), sites_only=shape == "sites_only", pad=shape == "one")
    sample, extra = ("NEW", ["--vcf-sample", "NEW"]) if shape == "sites_only" else (None, [])
    path = tmp_path / "in.vcf"
    path.write_text(text)
    env = dict(os.environ, **({"BRC_CLI_DEVICE_DECODE": "1"} if shape == "device_decode" else {}))
    sl = tmp_path / "derived"
    sl.write_text(complex_rule.derive(text))
    want = subprocess.run([exe] + argv + ["-f", fa, "-l", str(sl), bam], capture_output=True, env=env)
    got = subprocess.run([exe] + argv + extra + ["-f", fa, "--vcf", str(path), "--vcf-complex", bam], capture_output=True, env=env)
    plain = subprocess.run([exe] + argv + extra + ["-f", fa, "--vcf", str(path), bam], capture_output=True, env=env)
    assert want.returncode == 0 and got.returncode == 0 and plain.returncode == 0, got.stderr.decode()[-2000:]
    assert got.stderr == want.stderr
    contigs = {"21"}
    expect = complex_rule.annotate(text, want.stdout.decode("latin-1"), _testbam_answers(text, fl), sample=sample, contigs=contigs)
    assert got.stdout.decode("latin-1") == expect
    # every record the complex rule does not take keeps plain --vcf's bytes
    g, p = got.stdout.decode().splitlines(), plain.stdout.decode().splitlines()
    assert len(g) == len(p)
    n_cx = 0
    for a, b in zip(g, p):
        if a.startswith("#"):
            assert a == b
            continue
        c = a.split("\t")
        if complex_rule.complex_alleles(int(c[1]), c[3], c[4].split(",")) is None or c[0] != "21":
            assert a == b
        else:
            n_cx += 1
    assert n_cx >= 20


def test_cli_crafted(tmp_path):
    samtools = cases.samtools()
    exe = cases.cli()
    bam, fa = complex_cases.write_crafted(str(tmp_path), samtools)
    os.mkdir(tmp_path / "decoded")
    case = complex_cases.crafted_case(str(tmp_path / "decoded"))
    recs = complex_cases.crafted_records()
    text = vcf_cases.vcf_text(recs)
    path = tmp_path / "c.vcf"
    path.write_text(text)
    sl = tmp_path / "derived"
    sl.write_text(complex_rule.derive(text))
    for argv, fl in CLI_FLAGS.values():
        want = subprocess.run([exe] + argv + ["-f", fa, "-l", str(sl), bam], capture_output=True)
        got = subprocess.run([exe] + argv + ["-f", fa, "--vcf", str(path), "--vcf-complex", bam], capture_output=True)
        assert got.returncode == 0 and got.stderr == want.stderr, got.stderr.decode()
        ans = complex_cases.rule_answers(case, recs, fl)
        expect = complex_rule.annotate(text, want.stdout.decode(), lambda ch, p0, n, al: ans[(p0, n, tuple(al))], contigs={"chr1"})
        assert got.stdout.decode() == expect


def test_cli_vcf_samples_columns_equal_single_runs(tmp_path):
    exe = cases.cli()
    fa = cases.write_testbam_fasta(str(tmp_path / "ref.fa"))
    bam = os.path.join(cases.GOLDEN, "test.bam")
    text = vcf_cases.vcf_text(vcf_cases.fixture_records(), samples=("S1", "S2"))
    path = tmp_path / "in.vcf"
    path.write_text(text)
    lst = tmp_path / "samples"
    lst.write_text(f"S2\t{bam}\nS1\t{bam}\n")
    both = subprocess.run([exe, "-q", "20", "-f", fa, "--vcf", str(path), "--vcf-complex", "--vcf-samples", str(lst)], capture_output=True)
    assert both.returncode == 0, both.stderr.decode()
    cols = {}
    for s in ("S1", "S2"):
        one = subprocess.run([exe, "-q", "20", "-f", fa, "--vcf", str(path), "--vcf-complex", "--vcf-sample", s, bam], capture_output=True)
        assert one.returncode == 0
        k = 9 if s == "S1" else 10
        cols[s] = [ln.split("\t")[k] for ln in one.stdout.decode().splitlines() if ln and not ln.startswith("#")]
    rows = [ln.split("\t") for ln in both.stdout.decode().splitlines() if ln and not ln.startswith("#")]
    assert [r[9] for r in rows] == cols["S1"] and [r[10] for r in rows] == cols["S2"]
    assert any(":" in c and c.split(":")[2] not in (".", "0") for c in cols["S1"])
