"""Entry bounds of the alternative-allele site filter (brc_set_site_filter_bounds, Engine.set_site_filter(bounds=...),
brc-readcount --alt-min / --alt-max).

The rule is defined on the text (tests/alt_bounds_rule.py): a filtered run prints exactly select_lines_bounds of the unfiltered
output.
CPU: the rule on hand-written lines and on every committed golden, the hundredths routine against printf, the exact conversion
of Python bounds, CLI refusals and usage, the exported symbol.
GPU: engine and CLI output against the rule applied to the oracle's text and to the unfiltered run, device selection exactness,
rounding at a threshold, argv regions with the carried deletion queue, the pipelined, device-resident and pool-overflow paths,
and bounds that change nothing.
"""
import os
import re
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import cases
import golden_jobs
from alt_bounds_rule import FIELDS, FPFILTER_SETS, entries, line_passes_bounds, one_sided_sets, select_lines_bounds
from cases import GOLDEN, crafted_case, first_diff
from cases import cli as _cli
from site_filter_rule import is_alt, select_lines


def _printed(bounds):
    """{name: (lo, hi)} in hundredths -> the same in printed units (decimal strings) for Engine.set_site_filter."""
    f = lambda x: None if x is None else f"{x // 100}.{x % 100:02d}"
    return {k: (f(lo), f(hi)) for k, (lo, hi) in bounds.items()}


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
_ZERO = [0] * 13


def _ent(allele, v):
    """An entry string from 13 values in hundredths (integer fields printed as integers)."""
    ints = {0, 4, 5, 9}
    return allele + "".join(":" + (str(x // 100) if k in ints else f"{x // 100}.{x % 100:02d}") for k, x in enumerate(v))


def _line(ref, depth, *ents, libs=None):
    if libs:
        body = "".join(f"\t{lib}\t{{\t" + "\t".join(es) + "\t}" for lib, es in libs)
    else:
        body = "\t" + "\t".join(ents)
    return f"chr1\t100\t{ref}\t{depth}{body}"


def _base_entries(ref_count=5, alt=None):
    es = [_ent(b, _ZERO) for b in "=ACGTN"]
    es[1] = _ent("A", [ref_count * 100] + _ZERO[1:])
    if alt is not None:
        es[2] = _ent("C", alt)
    return es


def test_rule_each_field_at_its_bound_and_one_hundredth_off():
    v = [700, 3012, 2750, 1999, 400, 300, 45, 3, 1525, 200, 1233, 1, 8761]
    ln = _line("A", 12, *_base_entries(alt=v))
    assert [e[1] for e in entries(ln.split("\t")[4:])][2] == v
    for k, name in enumerate(FIELDS):
        x = v[k]
        assert line_passes_bounds(ln, 1, 0.0, {name: (x, None)}) and line_passes_bounds(ln, 1, 0.0, {name: (None, x)})
        assert line_passes_bounds(ln, 1, 0.0, {name: (x - 1, None)}) and not line_passes_bounds(ln, 1, 0.0, {name: (x + 1, None)})
        assert line_passes_bounds(ln, 1, 0.0, {name: (None, x + 1)}) and not line_passes_bounds(ln, 1, 0.0, {name: (None, x - 1)})
        assert line_passes_bounds(ln, 1, 0.0, {name: (x, x)}) and not line_passes_bounds(ln, 8, 0.0, {name: (x, x)})


def test_rule_indel_basequality_library_blocks_and_deletions():
    ins = [300, 6000, 0, 6000, 300, 0, 50, 0, 0, 0, 0, 0, 4000]
    ln = _line("A", 8, *_base_entries(), _ent("+GT", ins))
    assert line_passes_bounds(ln, 1, 0.0, {"avg_basequality": (None, 0)})
    assert not line_passes_bounds(ln, 1, 0.0, {"avg_basequality": (1, None)})       # an indel prints 0.00
    lib0 = _base_entries(alt=[200, 6000, 3000, 6000, 200, 0] + [0] * 7)               # one strand only
    lib1 = _base_entries(alt=[200, 6000, 3000, 6000, 100, 100] + [0] * 7)
    both = {"num_plus_strand": (100, None), "num_minus_strand": (100, None)}
    per_lib = _line("A", 14, libs=[("lib0", lib0), ("lib1", lib1)])
    assert line_passes_bounds(per_lib, 2, 0.0, both)                                  # lib1's entry qualifies
    only0 = _line("A", 14, libs=[("lib0", lib0), ("lib1", lib0)])
    assert not line_passes_bounds(only0, 2, 0.0, both) and line_passes_bounds(only0, 2, 0.0, {})
    dele = _line("A", 6, *_base_entries(), _ent("-AC", [100, 300, 0, 300, 0, 100] + [0] * 7))
    assert line_passes_bounds(dele, 1, 0.0, {"avg_mapping_quality": (None, 300), "num_minus_strand": (100, None)})
    assert not line_passes_bounds(dele, 1, 0.0, {"avg_mapping_quality": (301, None)})
    assert not line_passes_bounds(_line("A", 6, *_base_entries(ref_count=6)), 1, 0.0, {})  # the reference base never counts


def test_rule_on_goldens_is_a_subsequence_and_a_direct_restatement():
    texts = cases.golden_texts()
    assert len(texts) >= 30
    for name, text in texts:
        lines = text.splitlines()
        for mc, mf, bounds in [(1, 0.0, b) for b in FPFILTER_SETS + one_sided_sets(text)[:6]] + [(2, 0.05, FPFILTER_SETS[0])]:
            kept = select_lines_bounds(text, mc, mf, bounds).splitlines()
            it = iter(lines)
            assert all(any(k == x for x in it) for k in kept), name
            keep = set(kept)
            for ln in lines:
                f = ln.split("\t")
                ok = False
                for fld in f[4:]:
                    p = fld.split(":")
                    if len(p) != 14 or not re.fullmatch(r"[=ACGTN]|[+-][^:]*", p[0]):
                        continue
                    vals = [round(float(x) * 100) for x in p[1:]]
                    ok |= (is_alt(p[0], f[2]) and int(p[1]) >= mc and int(p[1]) >= mf * int(f[3])
                           and all((lo is None or vals[FIELDS.index(n)] >= lo) and (hi is None or vals[FIELDS.index(n)] <= hi)
                                   for n, (lo, hi) in bounds.items()))
                assert (ln in keep) == ok, (name, bounds, ln[:160])
        assert select_lines_bounds(text, 1, 0.0, {}) == select_lines(text, 1)
        assert select_lines_bounds(text, 1, 0.0, {n: (0, None) for n in FIELDS}) == select_lines(text, 1)


def test_hundredths_routine_matches_printf():
    p = subprocess.run([cases.check_program("hundredths_check", "-pthread")], capture_output=True, text=True)
    assert p.returncode == 0 and " 0 mismatches" in p.stdout, p.stdout[-2000:]


def test_python_bounds_convert_exactly():
    from decimal import Decimal
    from bam_readcount_b200.engine import entry_bounds, hundredths
    assert hundredths("0.29") == 29 and hundredths(0.29) == 29 and hundredths(Fraction(29, 100)) == 29   # 0.29 * 100 != 29.0
    assert hundredths(Decimal("12.5")) == 1250 and hundredths(7) == 700 and hundredths("1") == 100
    for bad in ("0.125", "-1", "x", "nan", -0.5, Fraction(1, 3), True):
        with pytest.raises(ValueError):
            hundredths(bad)
    b = entry_bounds({"num_minus_strand": ("1", None), "avg_basequality": (None, "20.05")})
    assert b.lo_set == 1 << 5 and b.hi_set == 1 << 2 and b.lo[5] == 100 and b.hi[2] == 2005
    with pytest.raises(ValueError):
        entry_bounds({"strand": (1, None)})


def test_cli_bound_refusals_and_usage():
    exe = _cli()
    bam = os.path.join(GOLDEN, "test.bam")
    env = dict(os.environ, BRC_CLI_DECODE_ONLY="1")
    for bad, msg in ((["--alt-min", "strand=1"], b"--alt-min"), (["--alt-max", "count=1.234"], b"--alt-max"),
                     (["--alt-min", "count=-1"], b"--alt-min"), (["--alt-min", "count=1."], b"--alt-min"),
                     (["--alt-min", "count=.5"], b"--alt-min"), (["--alt-min", "count"], b"--alt-min"),
                     (["--alt-min", "count=1e3"], b"--alt-min"), (["--alt-max", "count="], b"--alt-max"),
                     (["--alt-min", "count=1", "--alt-min", "count=2"], b"--alt-min"),
                     (["--alt-min", "avg_basequality=20.01", "--alt-max", "avg_basequality=20"], b"--alt-min")):
        p = subprocess.run([exe] + bad + [bam, "21:10402985-10402990"], capture_output=True, env=env)
        assert p.returncode == 1 and msg in p.stderr, (bad, p.stderr)
    p = subprocess.run([exe, "--alt-max", "count=9", "--vcf", os.path.join(GOLDEN, "absent.vcf"), bam], capture_output=True, env=env)
    assert p.returncode == 1 and b"--vcf cannot be combined with --alt-min/--alt-max" in p.stderr, p.stderr
    for good in (["--alt-min", "count=2"], ["--alt-max", "avg_pos_as_fraction=0.9", "--alt-min", "avg_pos_as_fraction=0.1"],
                 ["--alt-min", "avg_basequality=20", "--alt-max", "avg_basequality=20", "--min-alt-count", "2"]):
        p = subprocess.run([exe] + good + [bam, "21:10402985-10402990"], capture_output=True, env=env)
        assert p.returncode == 0, (good, p.stderr)
    p = subprocess.run([exe, "-h"], capture_output=True)
    assert b"--alt-min NAME=V" in p.stdout and b"--alt-max NAME=V" in p.stdout
    assert all(n.encode() in p.stdout.replace(b"\n", b"").replace(b" ", b"") for n in FIELDS)


def test_bounds_symbol_is_exported():
    from bam_readcount_b200 import build, engine
    build.build()
    lib = engine.load_library()
    assert hasattr(lib, "brc_set_site_filter_bounds") and "brc_set_site_filter_bounds" in engine.EXPORTS
    assert lib.brc_abi_version() == 2


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
def _runs(case, flags, site_list, filters, *, carry=False):
    """One engine, one batch per filter: [(text, selected, launches)] for each (min_alt_count, min_alt_fraction, bounds in
    hundredths or None; None = no filter).  carry: one compute per region with the deletion queue carried (brc-readcount's way)."""
    out = []
    with cases.open_engine(case, flags) as e:
        for filt in filters:
            if filt is None:
                e.clear_site_filter()
            else:
                mc, mf, b = filt
                e.set_site_filter(mc, mf, bounds=None if b is None else _printed(b))
            if carry:
                e.set_queue_carry(True)
                text = ""
                for region in case["regions"]:
                    e.reset()
                    cases.push_regions(e, case, site_list, [region])
                    e.compute()
                    text += e.format_text(-1)
                e.set_queue_carry(False)
                out.append((text, None, e.launch_count()))
                continue
            e.reset()
            cases.push_regions(e, case, site_list)
            res = e.compute()
            out.append((e.format_text(-1), e.selected() if res is None else None, e.launch_count()))
    return out


def _bound_sets(text):
    return one_sided_sets(text) + FPFILTER_SETS + [{n: (0, None) for n in FIELDS}]


_JOBS = [j for j in golden_jobs.jobs() if j[0].startswith(("syn-", "deep-", "edge-fuzz", "testbam-"))
         and not any(j[0].endswith(s) for s in ("perlib_ic_q20b20", "perlib_ic_q20"))]


@pytest.mark.gpu
@pytest.mark.parametrize("job", _JOBS, ids=[j[0] for j in _JOBS])
def test_engine_bounded_text_equals_the_rule_on_the_oracle_text(job):
    """Per field a min and a max bound at a value an alternative entry prints, three fpfilter-like sets and all-min-0, at
    count 1 and at (2, 0.05); the unfiltered run equals the oracle's text.  Site lists and single-region syn- cases: the device's
    emit-1 sites are exactly the rule's lines."""
    name, getter, flags, site_list, golden = job
    case = getter()
    want_all = cases.load_golden_text(golden)
    sets = _bound_sets(want_all)
    assert len(sets) >= 2 * 12 + 4
    filters = [None] + [(1, 0.0, b) for b in sets] + [(2, 0.05, b) for b in FPFILTER_SETS]
    runs = _runs(case, flags, site_list, filters)
    assert not first_diff(runs[0][0], want_all), first_diff(runs[0][0], want_all)
    exact = site_list or name.startswith("syn-")
    for filt, (text, sel, _) in zip(filters[1:], runs[1:]):
        want = select_lines_bounds(want_all, *filt)
        d = first_diff(text, want)
        assert not d, (filt, d)
        if exact:
            assert [p + 1 for p in sel.positions(1)] == [int(ln.split("\t")[1]) for ln in want.splitlines()], filt
    n_min0 = filters.index((1, 0.0, {n: (0, None) for n in FIELDS}))
    assert runs[n_min0][0] == select_lines(want_all, 1)


@pytest.mark.gpu
def test_rounding_at_the_threshold_and_on_binary_ties():
    """Eight reads with Σmapq 1 carry an alternative base at 101 (mean 0.125, printed 0.12), eight with Σmapq 3 one at 121 (0.375,
    printed 0.38): a bound equal to the printed value passes, one hundredth beyond it does not."""
    reads = [(80, "60M", set(), 0, 60, 0) for _ in range(10)]
    reads += [(90, "40M", {100}, 0, 1 if k == 0 else 0, 16 * (k & 1)) for k in range(8)]
    reads += [(110, "40M", {120}, 0, 1 if k < 3 else 0, 0) for k in range(8)]
    case = crafted_case(reads, [(0, 81, 140)])
    want, _, _ = cases.run_oracle(case, dict(), site_list=False)
    mq = {int(ln.split("\t")[1]): [v[1] for a, v in entries(ln.split("\t")[4:]) if is_alt(a, ln.split("\t")[2]) and v[0] > 0]
          for ln in want.splitlines()}
    assert mq[101] == [12] and mq[121] == [38]
    checks = [({"avg_mapping_quality": (12, None)}, [101, 121]), ({"avg_mapping_quality": (13, None)}, [121]),
              ({"avg_mapping_quality": (None, 12)}, [101]), ({"avg_mapping_quality": (None, 11)}, []),
              ({"avg_mapping_quality": (38, 38)}, [121]), ({"avg_mapping_quality": (39, None)}, []),
              ({"avg_mapping_quality": (None, 37)}, [101])]
    runs = _runs(case, dict(), False, [(1, 0.0, b) for b, _ in checks])
    for (b, sites), (text, _, _) in zip(checks, runs):
        assert [int(ln.split("\t")[1]) for ln in text.splitlines()] == sites, b
        assert text == select_lines_bounds(want, 1, 0.0, b), b


@pytest.mark.gpu
@pytest.mark.parametrize("carry", [False, True], ids=["one_batch", "carried_queue"])
def test_argv_regions_deletion_from_an_earlier_region_judged_by_its_stats(carry):
    """-p, argv regions Z, A, B = Z again (the carried-queue case of test_site_filter.py), with the deletion read of library 1
    on the minus strand at mapq 30 and every other read on the plus strand at mapq 60: bounds on strand or mapping quality make
    the deletion the only qualifying entry, or disqualify it, on the lines the host forms from the queue."""
    reads = [(30, "100M", {50} if k < 3 else set(), 0, 60, 0) for k in range(20)]
    reads += [(30, "50M", set(), 1, 60, 0) for _ in range(5)] + [(30, "30M1D19M", set(), 1, 30, 16)]
    case = crafted_case(reads, [(0, 41, 60), (0, 71, 120), (0, 41, 61)], n_libs=2)
    flags = dict(per_lib=True)
    want, _, _ = cases.run_oracle(case, flags, site_list=False)
    sets = [{"num_minus_strand": (100, None)}, {"num_minus_strand": (None, 0)}, {"avg_mapping_quality": (None, 3000)},
            {"avg_mapping_quality": (3001, None)}, {"avg_mapping_quality": (3000, 3000), "num_plus_strand": (None, 0)}]
    kept = [select_lines_bounds(want, 1, 0.0, b) for b in sets]
    assert [ln.split("\t")[1] for ln in kept[0].splitlines()] == ["61"] and "\t-" in kept[0]   # only the deletion's line
    assert kept[0] == kept[2] and [ln.split("\t")[1] for ln in kept[1].splitlines()] == ["51", "51"]
    runs = _runs(case, flags, False, [(1, 0.0, b) for b in sets] + [(2, 0.0, b) for b in sets], carry=carry)
    for filt, (text, _, _) in zip([(1, 0.0, b) for b in sets] + [(2, 0.0, b) for b in sets], runs):
        d = first_diff(text, select_lines_bounds(want, *filt))
        assert not d, (filt, d)


@pytest.mark.gpu
@pytest.mark.parametrize("n_chunks", [1, 7, 65])
def test_pipelined_path_with_bounds(n_chunks, monkeypatch):
    import pipeline_cases as pc
    case = pc.chunk_cuts(3)
    monkeypatch.setenv("BRC_PIPE_CHUNKS", str(n_chunks))
    for fname in ("default", "perlib"):
        otext = cases.run_oracle_cached(case, cases.FLAG_SETS[fname], False).text
        filters = [(1, 0.0, b) for b in FPFILTER_SETS + one_sided_sets(otext)[::5]]
        for filt, (text, _, _) in zip(filters, _runs(case, cases.FLAG_SETS[fname], False, filters)):
            d = first_diff(text, select_lines_bounds(otext, *filt))
            assert not d, (fname, n_chunks, filt, d)


@pytest.mark.gpu
def test_pool_overflow_fallback_with_bounds():
    import boundary_cases
    case = boundary_cases.pool_case()
    want = cases.run_oracle(case, dict(), site_list=True).text
    filters = [(1, 0.0, b) for b in FPFILTER_SETS + one_sided_sets(want)[:4]]
    for filt, (text, _, _) in zip(filters, _runs(case, dict(), True, filters)):
        d = first_diff(text, select_lines_bounds(want, *filt))
        assert not d, (filt, d)


@pytest.mark.gpu
def test_device_resident_run_selects_exactly_the_rule_lines():
    """brc_plan_device / brc_run_device on reads already on the device, with bounds: the emit-1 sites are the rule's lines of
    the oracle's text (a site list: nothing is carried in)."""
    import torch
    from bam_readcount_b200.engine import CRegion
    case = cases.synthetic_case(L=20000, depth=30, seed=29, regions=((0, 1, 20000),), site_list=True)
    want = cases.run_oracle(case, dict(), site_list=True).text
    region = case["regions"][0]
    tid, beg, end, sub, first_pos, n_slots, _ = cases.region_geometry(case, region)
    dev = torch.device("cuda", 0)
    cb, keep = cases.device_batch(sub, dev)
    with cases.open_engine(case) as e:
        s = torch.cuda.Stream(device=dev)
        for b in FPFILTER_SETS + one_sided_sets(want)[::4]:
            e.set_site_filter(1, 0.0, bounds=_printed(b))
            e.plan_device([CRegion(tid, beg, end, 1, 0, sub.n_reads, 0, first_pos, n_slots)], sub.n_reads, 1 << 20)
            e.run_device(cb, None, s.cuda_stream)
            assert e.fetch_device_results(s.cuda_stream) is None
            got = [p + 1 for p in e.selected().positions(1)]
            assert got == [int(ln.split("\t")[1]) for ln in select_lines_bounds(want, 1, 0.0, b).splitlines()], b
    del keep


@pytest.mark.gpu
def test_absent_or_always_true_bounds_change_nothing():
    """All-min-0 bounds give the text of the filter without bounds; bounds=None (brc_set_site_filter_bounds(f, NULL)) gives
    its text and launch count; a later filter without bounds has cleared them."""
    import ctypes as C
    from bam_readcount_b200.engine import BrcError, CEntryBounds, CSiteFilter
    case = cases.synthetic_case(L=30000, depth=30, seed=31, regions=((0, 1, 30000),), site_list=False)
    for flags in (dict(), dict(per_lib=True, insertion_centric=True)):
        plain = cases.run_engine(case, flags, False, dump=False, site_filter=(2, 0.05))
        with cases.open_engine(case, flags) as e:
            f = CSiteFilter(2, 0, 0.05)
            results = []
            for how in ("null", "zero", "min0", "cleared"):
                if how == "null":
                    e._check(e.lib.brc_set_site_filter_bounds(e.h, C.byref(f), None))
                elif how == "zero":
                    e._check(e.lib.brc_set_site_filter_bounds(e.h, C.byref(f), C.byref(CEntryBounds())))
                elif how == "min0":
                    e.set_site_filter(2, 0.05, bounds={n: (0, None) for n in FIELDS})
                else:
                    e.set_site_filter(2, 0.05, bounds={"count": (10 ** 6, None)})
                    e.set_site_filter(2, 0.05)
                e.reset()
                cases.push_regions(e, case, False)
                e.compute()
                results.append((how, e.format_text(-1), e.launch_count()))
            for how, text, launches in results:
                assert text == plain.text, (flags, how, first_diff(text, plain.text))
                assert launches == plain.launches, (flags, how)
            b = CEntryBounds()
            for bad in ("nofilter", "mask", "neg", "order"):
                b = CEntryBounds()
                if bad == "mask":
                    b.lo_set = 1 << 13
                elif bad == "neg":
                    b.hi_set, b.hi[3] = 1 << 3, -1
                elif bad == "order":
                    b.lo_set = b.hi_set = 1 << 6
                    b.lo[6], b.hi[6] = 51, 50
                rc = e.lib.brc_set_site_filter_bounds(e.h, None if bad == "nofilter" else C.byref(f), C.byref(b))
                assert rc != 0, bad
            with pytest.raises(BrcError):
                e.set_site_filter(2, 0.05, bounds={"avg_basequality": ("20", "19.99")})


def _cli_args(bounds):
    out = []
    for n, (lo, hi) in bounds.items():
        for opt, x in (("--alt-min", lo), ("--alt-max", hi)):
            if x is not None:
                out += [opt, f"{n}={x // 100}.{x % 100:02d}" if x % 100 else f"{n}={x // 100}"]
    return out


def _check_cli(exe, argv):
    full = subprocess.run([exe] + argv, capture_output=True)
    assert full.returncode == 0, full.stderr.decode()[-2000:]
    text = full.stdout.decode("latin-1")
    sets = FPFILTER_SETS + one_sided_sets(text)[::9]
    for i, b in enumerate(sets):
        for extra, mc in (([], 1), (["--min-alt-count", "2"], 2))[:1 if i else 2]:
            p = subprocess.run([exe] + extra + _cli_args(b) + argv, capture_output=True)
            assert p.returncode == 0, p.stderr.decode()[-2000:]
            d = first_diff(p.stdout.decode("latin-1"), select_lines_bounds(text, mc, 0.0, b))
            assert not d, (argv, b, extra, d)
            assert p.stderr == full.stderr
    return text


@pytest.mark.gpu
def test_cli_bounds_on_the_reference_fixture_and_a_synthetic_bam(tmp_path):
    exe = _cli()
    ref = cases.write_testbam_fasta(str(tmp_path / "ref.fa"))
    bam = os.path.join(GOLDEN, "test.bam")
    _check_cli(exe, ["-w", "0", "-f", ref, "-l", os.path.join(GOLDEN, "site_list"), bam])
    _check_cli(exe, ["-w", "0", "-p", "-f", ref, bam, "21:10402700-10403100", "21:10402950-10403300", "21:10403301-10403600"])
    from bam_readcount_b200 import synth
    case = cases.synthetic_case(L=30000, depth=30, seed=53, regions=((0, 1, 30000),), site_list=False)
    name, L, seq, _ = case["contigs"][0]
    d = str(tmp_path)
    synth.write_fasta(os.path.join(d, "s.fa"), name, np.frombuffer(seq, dtype=np.uint8))
    cases.write_bam(d, "s", case["batch"], [(name, L)], n_libs=len(case["lib_names"]))
    base = ["-w", "0", "-f", os.path.join(d, "s.fa"), os.path.join(d, "s.bam")]
    text = _check_cli(exe, base + ["chr1:1-30000"])
    assert any("\t+" in ln for ln in text.splitlines()) and any("\t-" in ln for ln in text.splitlines())
    _check_cli(exe, ["-p", "-i"] + base + ["chr1:1-12000", "chr1:11000-20000"])
    # --bam-list: each OUT equals that sample's single run with the same options
    lst = tmp_path / "list"
    runs = {"o1": (os.path.join(d, "s.fa"), os.path.join(d, "s.bam"), "chr1:1-30000"), "o2": (ref, bam, "21:10402700-10403100")}
    for b in FPFILTER_SETS[:1]:
        opts = _cli_args(b) + ["-p", "-w", "0"]
        for o, (fa, path, region) in runs.items():
            single = subprocess.run([exe] + opts + ["-f", fa, path, region], capture_output=True)
            assert single.returncode == 0
            lst.write_text(f"{path}\t{d}/{o}\n")
            p = subprocess.run([exe] + opts + ["-f", fa, "--bam-list", str(lst), region], capture_output=True)
            assert p.returncode == 0, p.stderr.decode()[-2000:]
            with open(os.path.join(d, o), "rb") as fh:
                assert fh.read() == single.stdout, (o, b)
