"""CPU: the C-ABI shared library builds, loads and exports every symbol include/brc_engine.h
declares; without a GPU it refuses to create an engine (no CPU fallback)."""
import os
import re

import pytest

from cases import ROOT


def _declared():
    txt = open(os.path.join(ROOT, "include", "brc_engine.h")).read()
    return sorted(set(re.findall(r"BRC_API[^;(]*?\b(brc_\w+)\s*\(", txt)))


def test_library_builds_and_exports_every_declared_symbol():
    from bam_readcount_b200 import build, engine
    build.build()
    lib = engine.load_library()
    decl = _declared()
    assert len(decl) >= 20
    for s in decl:
        assert hasattr(lib, s), f"{s} declared in include/brc_engine.h but not exported"
    assert sorted(engine.EXPORTS) == decl
    assert lib.brc_abi_version() == 2


def test_no_cpu_fallback_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from bam_readcount_b200 import engine
    with pytest.raises(engine.BrcError) as ei:
        engine.Engine()
    assert ei.value.status == -2   # BRC_E_NO_DEVICE


def test_product_never_imports_oracle():
    """The oracle is test infrastructure: nothing under the product package may import, include or run it."""
    pkg = os.path.join(ROOT, "bam_readcount_b200")
    bad = re.compile(r"(^\s*(from|import)\s+oracle\b)|(#include\s*[\"<][^\">]*oracle)|(oracle/_ref)|(liboracle)|(brc_oracle\.c\b.*(open|CDLL|subprocess))", re.M)
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                src = open(os.path.join(dp, f), errors="ignore").read()
                assert not bad.search(src), f"{f} reaches into oracle/"


def test_missing_extension_fails_loudly():
    """No silent fallback: asking for a library that is not there raises, with the build hint."""
    from bam_readcount_b200 import engine
    with pytest.raises(RuntimeError) as ei:
        engine.load_library("/nonexistent/libbrc_engine.so")
    assert "no CPU fallback" in str(ei.value)
