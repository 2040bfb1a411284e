"""In-tree build of libbrc_engine.so for sm_90a (H100) (explicit nvcc; no JIT cache, no torch)."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libbrc_engine.so")
SOURCES = ["brc_kernels.cu", "brc_engine.cu", "brc_bgzf.cu", "brc_select.cu", "brc_format.cpp"]
HEADERS = ["brc_device.cuh", "brc_engine_internal.h", "brc_fmt_num.h", "brc_aux.cuh", "brc_bgzf.cuh", "brc_scan.cuh", os.path.join("..", "..", "include", "brc_engine.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "--fmad=false",            # bit-exact float parity with the CPU reference: never contract a*b+c
    "-Xcompiler", "-fPIC,-O2,-Wall,-fvisibility=hidden",
    "-Xptxas", "-v",
    "-shared",
]


def nvcc_path() -> str:
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(p):
        raise RuntimeError("nvcc not found")
    return p


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    for f in SOURCES + HEADERS:
        if os.path.getmtime(os.path.join(CSRC, f)) > t:
            return True
    return os.path.getmtime(os.path.abspath(__file__)) > t


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    extra = os.environ.get("BRC_NVCC_EXTRA", "").split()
    cmd = [nvcc_path()] + NVCC_FLAGS + extra + ["-I", os.path.join(HERE, "..", "include"), "-o", LIB] + \
          [os.path.join(CSRC, s) for s in SOURCES]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if verbose or p.returncode != 0:
        sys.stderr.write(p.stdout)
    if p.returncode != 0:
        raise RuntimeError("nvcc failed building libbrc_engine.so")
    with open(os.path.join(HERE, "build.log"), "w") as fh:
        fh.write(" ".join(cmd) + "\n" + p.stdout)
    return LIB


def build_profile_variant(define: str = "-DBRC_DEEP_PROFILE") -> str:
    """An instrumented copy of the library (cycle counters inside a kernel) next to the product: libbrc_engine_prof.so.
    Loaded by the tools with BRC_ENGINE_LIB=<path>; never by the tests or the bench."""
    out = os.path.join(HERE, "libbrc_engine_prof.so")
    cmd = [nvcc_path()] + NVCC_FLAGS + [define, "-I", os.path.join(HERE, "..", "include"), "-o", out] + \
          [os.path.join(CSRC, s) for s in SOURCES]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout)
        raise RuntimeError("nvcc failed building libbrc_engine_prof.so")
    return out


SYNTH_LIB = os.path.join(HERE, "libbrc_synth.so")


def build_synth(force: bool = False) -> str:
    """The counter-based workload generator (include/brc_synth.h): device kernels + the identical host implementation."""
    src = os.path.join(CSRC, "brc_synth.cu")
    hdr = os.path.join(HERE, "..", "include", "brc_synth.h")
    if not force and os.path.exists(SYNTH_LIB) and os.path.getmtime(SYNTH_LIB) >= max(os.path.getmtime(src), os.path.getmtime(hdr)):
        return SYNTH_LIB
    flags = [f for f in NVCC_FLAGS if f != "--fmad=false"]
    cmd = [nvcc_path()] + flags + ["-I", os.path.join(HERE, "..", "include"), "-o", SYNTH_LIB, src]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout)
        raise RuntimeError("nvcc failed building libbrc_synth.so")
    return SYNTH_LIB


CLI = os.path.join(HERE, "brc-readcount")


def build_cli(force: bool = False) -> str:
    """The C++ host binary (same CLI / STDOUT as bam-readcount) on top of libbrc_engine.so."""
    src = os.path.join(CSRC, "brc_cli.cpp")
    hts_a = os.path.join(HERE, "third_party", "htslib", "libhts.a")
    newest = max([os.path.getmtime(src), os.path.getmtime(os.path.join(CSRC, "brc_aux.cuh")), os.path.getmtime(LIB)] + ([os.path.getmtime(hts_a)] if os.path.exists(hts_a) else []))
    if not force and os.path.exists(CLI) and os.path.getmtime(CLI) >= newest:
        return CLI
    cmd = ["g++", "-O2", "-std=c++17", "-Wall", "-o", CLI, src, "-I", os.path.join(HERE, "..", "include"),
           "-L", HERE, "-lbrc_engine"]
    hts = os.path.join(HERE, "third_party", "htslib")          # tools/build_htslib.sh: htslib 1.10 as vendored with the reference (CRAM only)
    if os.path.exists(os.path.join(hts, "libhts.a")):
        cmd += ["-DBRC_WITH_HTSLIB", "-I", hts, os.path.join(hts, "libhts.a"), "-lpthread"]
    cmd += ["-lz", "-Wl,-rpath,$ORIGIN"]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout)
        raise RuntimeError("g++ failed building brc-readcount")
    return CLI


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
    print(build_synth(force="--force" in sys.argv))
    print(build_cli(force="--force" in sys.argv))
