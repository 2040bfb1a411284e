"""Differential fuzz on seeds of their own (not the edge cases of tests/edge_cases.py):
  CPU: the oracle against what the unmodified reference binary printed for the same site lists (the SHA-256 of its STDOUT per
       seed and flag set, tests/golden/fresh_fuzz_sha256.json, written by tests/golden/make_golden.py) — pins the restatement on random CIGARs (D/N/=/X/H/P, P-then-I, leading
       deletions), missing NM/SM tags, filtered flags, reads without a library, -q/-b/-i/-p/-d.
  GPU: the engine against the oracle on the same cases, raw accumulators bit-for-bit, with and without the deep-site kernel
       forced onto the small tiles."""
import numpy as np
import pytest

import cases
from edge_cases import FRESH_SEEDS as SEEDS
from edge_cases import fresh_fuzz_case as _case


@pytest.mark.parametrize("seed", SEEDS)
def test_oracle_equals_reference_binary_on_fresh_fuzz(seed):
    case = _case(seed)
    for fname, fl in case["flag_sets"].items():
        cases.assert_anchor("fresh_fuzz_sha256.json", f"{seed}_{fname}", cases.run_oracle(case, fl, site_list=True).text)


@pytest.mark.gpu
@pytest.mark.parametrize("deep", (False, True), ids=("pileup", "deep-forced"))
@pytest.mark.parametrize("seed", SEEDS)
def test_engine_equals_oracle_on_fresh_fuzz(seed, deep, monkeypatch):
    if deep:
        monkeypatch.setenv("BRC_DEEP_MIN_READS", "1")
    case = _case(seed)
    # single-base site-list lines as well as the whole contig: the small tiles are what the deep-site kernel takes
    L = case["contigs"][0][1]
    rng = np.random.default_rng(seed + 1000)
    case = dict(case, regions=[(0, 1, L)] + [(0, int(p), int(p)) for p in np.sort(rng.integers(2, L - 2, 25))])
    for fname, fl in case["flag_sets"].items():
        cases.assert_same(cases.run_engine(case, fl, site_list=True), cases.run_oracle(case, fl, site_list=True), fname)
