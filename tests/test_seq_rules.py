"""CPU: htslib's base-code and CIGAR rules as brc_seq.cuh states them for the kernels, the engine host and brc-readcount, against
the oracle's independent C definitions (tests/seq_check.cpp, compiled with g++): the seq_nt16 table for all 256 bytes, the
canonical table for all 16 codes, and bam_endpos from cigar_span on every read of the committed BAM fixtures, of the crafted
complex-record BAM and of random CIGARs over every op."""
import os
import subprocess

import numpy as np
import pytest

import cases
import complex_cases
from bam_readcount_b200 import bamio


@pytest.fixture(scope="module")
def seq_check():
    return cases.check_program("seq_check")


def test_tables_equal_oracle(seq_check):
    p = subprocess.run([seq_check, "tables"], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout[:2000]
    assert p.stdout.split() == ["ok", str(256 + 3 * 16 + 256 * 4)]


def _span_lines(reads):
    """(flag, pos, CIGAR words) of each read, once more as an unmapped read and once without CIGAR: the check program's input
    lines and the I/D op count of each."""
    lines, n_indel = [], []
    for flag, pos, cig in reads:
        for f, c in ((flag, cig), (flag | 4, cig), (flag & ~4, [])):
            lines.append(f"{f} {pos} {len(c)} " + " ".join(map(str, c)))
            n_indel.append(sum(1 for w in c if w & 15 in (1, 2)))
    return lines, n_indel


def _bam_reads(path):
    batch = bamio.read_bam(path)[1]
    return [(int(batch.flag[i]), int(batch.pos[i]), batch.cigar[int(batch.cigar_off[i]):int(batch.cigar_off[i + 1])].tolist())
            for i in range(batch.n_reads)]


def _random_reads(n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        k = int(rng.integers(1, 12))
        ops, lens = rng.integers(0, 10, k), rng.integers(0, 1 << 28, k) >> rng.integers(0, 28, k)
        out.append((int(rng.integers(0, 2048)), int(rng.integers(-1, 1 << 31)), [int(l) << 4 | int(o) for o, l in zip(ops, lens)]))
    return out


def test_cigar_span_equals_read_endpos(seq_check, tmp_path):
    reads = _bam_reads(os.path.join(cases.GOLDEN, "test.bam")) + _bam_reads(os.path.join(cases.GOLDEN, "test_bad_rg.bam"))
    reads += _bam_reads(complex_cases.write_crafted(str(tmp_path))[0]) + _random_reads(2000, 11)
    lines, n_indel = _span_lines(reads)
    out = subprocess.run([seq_check, "span"], input="\n".join(lines) + "\n", capture_output=True, text=True,
                         check=True).stdout.splitlines()
    assert len(out) == len(lines) > 6000
    got = [tuple(map(int, o.split())) for o in out]
    bad = [(lines[k], got[k]) for k in range(len(got)) if got[k][0] != got[k][1] or got[k][2] != n_indel[k]]
    assert not bad, bad[:5]
    assert sum(g[2] > 0 for g in got) > 1000
