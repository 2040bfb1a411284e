"""K0's output pinned byte for byte: the read descriptors and the tile ranges the pileup kernels read.

Each case runs through the engine once; the SHA-256 of its descriptors (80 bytes per read) followed by tile_lo and tile_hi is
compared with tests/golden/k0_descriptors.json.  The cases: a C4 window of the generator (bench.py's workload), every boundary
fixture (K0's stage capacities, the staged reference window, reads past it), the contigs of length near 2^31, and a synthetic case
under -q 20 -b 20 -p.  A change to K0 that keeps every ReadDesc field and every tile range keeps these hashes.

    python tests/test_k0_descriptors.py --write FILE     # writes the hashes of the library in this tree (needs a GPU)
"""
from __future__ import annotations

import functools
import hashlib
import json
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "k0_descriptors.json")
QBP = dict(min_mapq=20, min_bq=20, per_lib=True)


def _digest(desc, lo, hi) -> str:
    h = hashlib.sha256()
    for a in (desc, lo, hi):
        h.update(a.tobytes())
    return h.hexdigest()


def _fixture_digest(case, flags) -> str:
    import cases
    with cases.open_engine(case, flags) as e:
        cases.push_regions(e, case, case["modes"][0] if "modes" in case else case["site_list"])
        e.compute()
        return _digest(*e.read_descriptors())


def _c4_digest() -> str:
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
        return _digest(*r.eng.read_descriptors())
    finally:
        r.close()


@functools.lru_cache(maxsize=None)
def case_list():
    """{name: thunk returning the digest}"""
    import boundary_cases
    import cases
    import edge32_cases
    out = {"c4_window": _c4_digest}
    for c in boundary_cases.all_cases():
        for fname in ("default", "perlib_ic_q20b20"):
            out[f"{c['name']}_{fname}"] = functools.partial(_fixture_digest, c, boundary_cases.FLAG_SETS[fname])
    for k in (0, 3):
        c = edge32_cases.contig_end_2_31(k)
        out[c["name"]] = functools.partial(_fixture_digest, c, {})
        s = edge32_cases.site_lines(c)
        out[s["name"]] = functools.partial(_fixture_digest, s, {})
    syn = cases.synthetic_case(L=40000, depth=30, seed=31, regions=((0, 2000, 38000),), n_libs=4)
    out["synthetic_q20_b20_p"] = functools.partial(_fixture_digest, syn, QBP)
    return out


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


def test_golden_covers_every_case():
    assert sorted(_golden()) == sorted(case_list())


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(case_list()))
def test_k0_descriptors_equal_golden(name):
    assert case_list()[name]() == _golden()[name], name


if __name__ == "__main__":
    if len(sys.argv) != 3 or sys.argv[1] != "--write":
        sys.exit(__doc__)
    sys.path[:0] = [os.path.dirname(HERE), HERE]
    got = {name: go() for name, go in sorted(case_list().items())}
    with open(sys.argv[2], "w") as f:
        json.dump(got, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"{len(got)} digests -> {sys.argv[2]}")
