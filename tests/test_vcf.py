"""GPU: allele queries (brc_set_allele_queries) and `brc-readcount --vcf`.

Engine: for every printed site of a batch, every kind of query — the six bases, every insertion and deletion the dense
results hold, and lengths and bases they do not — is answered exactly as a lookup in the Results of the same batch computed
without queries, with the depth and the line of the text.  CLI: --vcf STDOUT is tests/vcf_rule.py applied to the STDOUT of
`-l <derived site list>`, and its STDERR is that run's."""
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import cases
import edge_cases
import vcf_cases
import vcf_rule
from bam_readcount_b200.batch import ReadBatch
from bam_readcount_b200.engine import KIND_DEL, KIND_INS, CRegion, admitted

pytestmark = pytest.mark.gpu

FLAGS = {"default": {}, "ic": dict(insertion_centric=True), "q20b20": dict(min_mapq=20, min_bq=20), "d5": dict(max_cnt=5)}


def _lookup(res, reads, refs, tid, slot, pos):
    bases, indels = res._keys(0, slot, pos, reads, refs, tid, 0)
    return bases, {al: st for _, al, st in indels}


def _queries_and_expect(res, text, reads, refs):
    """Every query kind at every printed site, and the expected answer of each: (queries, bases, stats, depth)."""
    lines = iter(text.splitlines())
    q, buf, want = [], b"", []
    zero = np.zeros(13, np.uint32)
    for g, rg in enumerate(res.regions):
        tid = rg["tid"]
        for s in range(rg["n_slots"]):
            pos, slot = rg["first_pos"] + s, rg["slot_base"] + s
            if not (rg["beg"] <= pos < rg["end"]) or res.ncover[0, slot] == 0:
                continue
            f = next(lines).split("\t")
            assert int(f[1]) == pos + 1
            depth = int(f[3])
            bases, ind = _lookup(res, reads, refs, tid, slot, pos)
            for k in range(6):
                q.append((g, pos, k, 0)); want.append((bases.get(k, zero), depth))
            ins = [a for a in ind if a[0] == "+"]
            lens = {len(a) - 1 for a in ins}
            for a in ins + ["+" + "A" * (n + 1) for n in sorted(lens)] + ["+" + "".join("C" if c != "C" else "G" for c in a[1:]) for a in ins] + ["+T"]:
                q.append((g, pos, KIND_INS | (len(a) - 1) << 8, len(buf))); buf += a[1:].encode()
                want.append((ind.get(a, zero), depth))
            dels = {}
            if s > 0:
                _, dind = _lookup(res, reads, refs, tid, slot - 1, pos - 1)
                dels = {len(a) - 1: st for a, st in dind.items() if a[0] == "-"}
            for n in sorted(set(dels) | {1, 2, max(dels, default=0) + 1}):
                q.append((g, pos, KIND_DEL | n << 8, 0)); want.append((dels.get(n, zero), depth))
    assert next(lines, None) is None
    return q, buf, want


def _check_answers(e, q, buf, want):
    ans = e.allele_answers()
    assert len(ans) == len(q)
    for i, (st, depth) in enumerate(want):
        assert ans[i]["line"] == 1 and ans[i]["depth"] == depth, (q[i], ans[i])
        assert (ans[i]["stats"] == st).all(), (q[i], ans[i]["stats"], st)


def _engine_check(case, flags, site_list, push="one"):
    with cases.open_engine(case, flags) as e:
        pushed = cases.push_regions(e, case, site_list, push=push)
        res = e.compute()
        text = e.format_text(-1)
        cnt = flags.get("max_cnt", 10_000_000)
        reads = ReadBatch.concat([sub.select(admitted(sub, tid, cnt)) for tid, sub in pushed])
        refs = {cases.case_tid(case, ci): (wb, seq) for ci, (_, _, seq, wb) in enumerate(case["contigs"])}
        q, buf, want = _queries_and_expect(res, text, reads, refs)
        assert q, "no printed site"
        launches = e.launch_count()
        e.reset()
        cases.push_regions(e, case, site_list, push=push)
        e.set_allele_queries(q, buf)
        assert e.compute() is None
        _check_answers(e, q, buf, want)
        assert e.launch_count() == launches + 2 and e.stage_ms(4) > 0.0


def _cases():
    syn = cases.synthetic_case(L=6000, depth=30, seed=11, regions=[(0, p, p) for p in range(400, 5600, 37)], site_list=True)
    return {"testbam": (cases.testbam_case(), True), "syn_sites": (syn, True),
            "syn_argv": (cases.synthetic_case(L=6000, depth=30, seed=12, regions=[(0, 300, 2300), (0, 2600, 2900)]), False),
            "deep": (cases.deep_case(n_sites=2, depth=2500), True), "alleles": (edge_cases.multi_allele_case(), True)}


CASES = _cases()


@pytest.mark.parametrize("flags", list(FLAGS))
@pytest.mark.parametrize("name", list(CASES))
def test_answers_equal_dense_lookup(name, flags):
    case, sl = CASES[name]
    _engine_check(case, dict(FLAGS[flags]), sl)


def test_answers_pipelined_chunks(monkeypatch):
    """One long borrowed region, streamed through the GPU in 7 chunks (compute_pipelined)."""
    monkeypatch.setenv("BRC_PIPE_CHUNKS", "7")
    case = cases.synthetic_case(L=30000, depth=30, seed=13, regions=[(0, 2000, 26000)])
    _engine_check(case, {}, False)


def test_answers_device_path():
    """brc_plan_device / brc_run_device leave the answers on the device; brc_fetch_device_results copies them."""
    import torch
    case = dict(cases.synthetic_case(L=8000, depth=30, seed=14, regions=[(0, 500, 7000)]), lib_names=[])
    region = case["regions"][0]
    with cases.open_engine(case) as e:
        cases.push_regions(e, case, True)
        res = e.compute()
        text = e.format_text(-1)
        tid, beg, end, sub, first_pos, n_slots, _ = cases.region_geometry(case, region)
        refs = {tid: (case["contigs"][0][3], case["contigs"][0][2])}
        q, buf, want = _queries_and_expect(res, text, sub.select(admitted(sub, tid, 10_000_000)), refs)
        cb, keep = cases.device_batch(sub, torch.device("cuda:0"))
        stream = torch.cuda.Stream()
        e.plan_device([CRegion(tid, beg, end, 1, 0, sub.n_reads, 0, first_pos, n_slots)], sub.n_reads, 1 << 20)
        e.set_allele_queries(q, buf)
        e.run_device(cb, None, stream.cuda_stream)
        assert e.fetch_device_results(stream.cuda_stream) is None
        _check_answers(e, q, buf, want)


def test_refusals_and_reset():
    import ctypes as C
    from bam_readcount_b200.engine import RESULTS_ANSWERS, RESULTS_DENSE, RESULTS_NONE, BrcError, CPackedResults, CResults
    case = cases.synthetic_case(L=6000, depth=20, seed=15, regions=[(0, 500, 1500)], n_libs=2)   # prints sites [499, 1500)
    with cases.open_engine(case, dict(per_lib=True)) as e:
        cases.push_regions(e, case, True)
        assert e.results_kind() == RESULTS_NONE
        with pytest.raises(BrcError):
            e.set_allele_queries([(0, 600, 1, 0)])
        assert e.results_kind() == RESULTS_NONE
    with cases.open_engine(case) as e:
        cases.push_regions(e, case, True)
        e.compute()
        assert e.results_kind() == RESULTS_DENSE
        plain_text, plain_launches = e.format_text(-1), e.launch_count()
    with cases.open_engine(case) as e:
        e.set_site_filter(1, 0.0)
        cases.push_regions(e, case, True)
        assert e.results_kind() == RESULTS_NONE
        with pytest.raises(BrcError):
            e.set_allele_queries([(0, 600, 1, 0)])
        e.clear_site_filter()
        for bad, bases in (([(1, 600, 1, 0)], b""), ([(0, 498, 1, 0)], b""), ([(0, 1500, 1, 0)], b""), ([(0, 600, 9, 0)], b""),
                           ([(0, 600, 1 | 1 << 8, 0)], b""), ([(0, 600, KIND_DEL, 0)], b""), ([(0, 600, KIND_INS | 2 << 8, 0)], b"AR"),
                           ([(0, 600, KIND_INS | 2 << 8, 1)], b"AC")):
            with pytest.raises(BrcError):
                e.set_allele_queries(bad, bases)
            assert e.results_kind() == RESULTS_NONE
        e.set_allele_queries([(0, 499, 1, 0), (0, 1499, KIND_INS | 2 << 8, 0)], b"AC")
        with pytest.raises(BrcError):
            e.set_site_filter(1, 0.0)
        assert e.results_kind() == RESULTS_NONE
        assert e.lib.brc_compute(e.h) == 0
        assert e.results_kind() == RESULTS_ANSWERS
        assert e.lib.brc_get_results(e.h, C.byref(CResults())) != 0
        assert e.lib.brc_get_packed_results(e.h, C.byref(CPackedResults())) != 0
        assert e.lib.brc_format_text(e.h, -1, e._names_arr, None, 0) < 0
        with pytest.raises(BrcError):
            e.selected()
        assert e.results_kind() == RESULTS_ANSWERS
        assert len(e.allele_answers()) == 2 and e.stage_ms(4) > 0.0
        e.set_allele_queries([(0, 499, 1, 0)])                  # queries of a next run drop the answers of the last one
        assert e.results_kind() == RESULTS_NONE and e.stage_ms(4) == 0.0
        with pytest.raises(BrcError):
            e.allele_answers()
        assert e.lib.brc_compute(e.h) == 0
        assert e.results_kind() == RESULTS_ANSWERS and len(e.allele_answers()) == 1
        e.reset()
        assert e.results_kind() == RESULTS_NONE
        assert e.stage_ms(4) == 0.0
        cases.push_regions(e, case, True)
        assert e.results_kind() == RESULTS_NONE
        e.compute()
        assert e.results_kind() == RESULTS_DENSE
        assert e.format_text(-1) == plain_text and e.launch_count() == plain_launches


# ---------------------------------------------------------------------------------------------------------------- CLI
def _cli_pair(exe, tmp, vcf_text_, bam, fa, flags, extra=(), env=None, name="in.vcf", bgzf=False, sample=None):
    path = os.path.join(tmp, name)
    if bgzf:
        vcf_cases.write_bgzf(path, vcf_text_.encode())
    else:
        open(path, "w").write(vcf_text_)
    sl = os.path.join(tmp, name + ".sites")
    open(sl, "w").write(vcf_rule.derive(vcf_text_))
    env = dict(os.environ, **(env or {}))
    want = subprocess.run([exe] + flags + ["-f", fa, "-l", sl, bam], capture_output=True, env=env)
    got = subprocess.run([exe] + flags + list(extra) + ["-f", fa, "--vcf", path, bam], capture_output=True, env=env)
    assert want.returncode == 0 and got.returncode == 0, got.stderr.decode()[-2000:]
    assert got.stderr == want.stderr
    missing = {ln.split(" ")[0] for ln in want.stderr.decode().splitlines() if " not found in bam file." in ln}
    contigs = {ln.split("\t")[0] for ln in vcf_text_.splitlines() if ln and ln[0] != "#"} - missing
    text = want.stdout.decode("latin-1")
    assert got.stdout.decode("latin-1") == vcf_rule.annotate(vcf_text_, text, sample=sample, contigs=contigs)
    return text


CLI_FLAGS = {"default": [], "ic": ["-i"], "q20b20": ["-q", "20", "-b", "20"], "w2": ["-w", "2"]}


@pytest.mark.parametrize("flags", list(CLI_FLAGS))
@pytest.mark.parametrize("shape", ["one", "multi", "sites_only", "bgzf", "device_decode"])
def test_cli_vcf_fixture(tmp_path, flags, shape):
    exe = cases.cli()
    fa = cases.write_testbam_fasta(str(tmp_path / "ref.fa"))
    recs = vcf_cases.fixture_records()
    sample, extra = None, []
    if shape == "multi":
        sample, extra = "S2", ["--vcf-sample", "S2"]
    if shape == "sites_only":
        sample, extra = "NEW", ["--vcf-sample", "NEW"]
    text = vcf_cases.vcf_text(recs, samples=("S1", "S2") if shape == "multi" else ("S1",), sites_only=shape == "sites_only",
                              pad=shape == "one")
    out = _cli_pair(exe, str(tmp_path), text, os.path.join(cases.GOLDEN, "test.bam"), fa, CLI_FLAGS[flags], extra,
                    env={"BRC_CLI_DEVICE_DECODE": "1"} if shape == "device_decode" else None, bgzf=shape == "bgzf", sample=sample)
    with open(os.path.join(cases.GOLDEN, "vcf_sha256.json")) as fh:
        pinned = json.load(fh)
    key = "fixture_" + ("default" if flags == "w2" else flags)
    assert hashlib.sha256(out.encode("latin-1")).hexdigest() == pinned[key], "-l derived differs from the reference binary"


def test_cli_vcf_synthetic_indels(tmp_path):
    """A synthetic BAM with indels; records from its own text, so most alleles are present."""
    from bam_readcount_b200 import synth
    exe = cases.cli()
    L = 20000
    ref = synth.synth_reference(L, 31)
    batch = synth.synth_reads(ref, 30, seed=31, n_libs=2)
    d = str(tmp_path)
    fa = os.path.join(d, "s.fa")
    synth.write_fasta(fa, "chr1", ref)
    bam = cases.write_bam(d, "s", batch, [("chr1", L)], n_libs=2, read_group=True)
    sites = os.path.join(d, "all")
    open(sites, "w").write("".join(f"chr1\t{p}\t{p}\n" for p in range(200, L - 200)))
    lines = subprocess.run([exe, "-f", fa, "-l", sites, bam], capture_output=True, check=True).stdout.decode().splitlines()
    recs = []
    r = ref.tobytes().decode()
    for ln in lines[::7]:
        f = ln.split("\t")
        p = int(f[1])
        ents = [x.split(":")[0] for x in f[10:]]
        alts = [b for b in "ACGT" if b != r[p - 1]][:2]
        recs.append(("chr1", p, r[p - 1], ",".join(alts + [r[p - 1] + e[1:] for e in ents if e[0] == "+"][:2])))
        for e in ents:
            if e[0] == "-":
                recs.append(("chr1", p - 1, r[p - 2] + e[1:], r[p - 2]))
    text = vcf_cases.vcf_text(recs)
    for flags in (["-w", "0"], ["-w", "0", "-i"], ["-w", "0", "-q", "20", "-b", "20"]):
        _cli_pair(exe, d, text, bam, fa, flags)
