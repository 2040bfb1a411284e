"""Micro known-answers from SURVEY.md Appendix E (generated with the reference binary during the survey):
hand-built reads on the 50 bp contig `c` = ACGT x12 + AC, region c:10-10, and the `-d` max-count table.
CPU: the oracle; GPU: the CUDA engine through the C ABI."""
import numpy as np
import pytest

import cases
from bam_readcount_b200.batch import BatchBuilder

REF = ("ACGT" * 12 + "AC").encode()


def _case(reads, regions=((0, 10, 10),)):
    bb = BatchBuilder()
    for r in reads:
        bb.add_sam(tid=0, flag=0, mapq=60, lib=0, sm=None, qname="r", **r)
    return dict(name="ka", contigs=[("c", 50, REF, 0)], batch=bb.build(), regions=list(regions), site_list=False, lib_names=["lib0"])


def _mut(seq, i, b):
    return seq[:i] + b + seq[i + 1:]


R20 = REF[:20].decode()
KNOWN = [
    (dict(pos=0, cigar="20M", seq=_mut(R20, 5, "T"), qual="I" * 20, nm=1), "C:1:60.00:40.00:60.00:1:0:0.90:0.05:40.00:1:0.45:20.00:0.45"),
    (dict(pos=0, cigar="5=1X14=", seq=_mut(R20, 5, "T"), qual="I" * 20, nm=1), "C:1:60.00:40.00:60.00:1:0:0.90:0.05:0.00:1:0.45:20.00:0.45"),
    (dict(pos=0, cigar="3S17M", seq="TTT" + REF[:17].decode(), qual="I" * 20, nm=0), "C:1:60.00:40.00:60.00:1:0:0.94:0.00:0.00:1:0.30:17.00:0.30"),
    (dict(pos=0, cigar="5H3S17M", seq="TTT" + REF[:17].decode(), qual="I" * 20, nm=0), "C:1:60.00:40.00:60.00:1:0:0.59:0.00:0.00:1:0.30:17.00:0.25"),
]
D_TABLE = {100: [20, 20, 20, 40, 40], 10: [10, 10, 10, 11, 11], 5: [5, 5, 5, 6, 6], 1: [1, 1, 1, 2, 2], 0: [1, 1, 1, 2, 2]}


def _block(text, allele="C"):
    line = text.strip().split("\n")[0].split("\t")
    assert line[:2] == ["c", "10"] and line[3] == "1"
    return [f for f in line[4:] if f.startswith(allele + ":")][0]


def _d_case():
    reads = [dict(pos=4, cigar="20M", seq=REF[4:24].decode(), qual="I" * 20, nm=0) for _ in range(20)] + \
            [dict(pos=7, cigar="20M", seq=REF[7:27].decode(), qual="I" * 20, nm=0) for _ in range(20)]
    return _case(reads, regions=((0, 5, 9),))


@pytest.mark.parametrize("k", range(len(KNOWN)))
def test_oracle_known_answers(k):
    read, want = KNOWN[k]
    text, _, _ = cases.run_oracle(_case([read]), dict())
    assert _block(text) == want


@pytest.mark.parametrize("d", sorted(D_TABLE))
def test_oracle_max_count_table(d):
    text, _, _ = cases.run_oracle(_d_case(), dict(max_cnt=d))
    assert [int(l.split("\t")[3]) for l in text.strip().split("\n")] == D_TABLE[d]


@pytest.mark.gpu
@pytest.mark.parametrize("k", range(len(KNOWN)))
def test_engine_known_answers(k):
    read, want = KNOWN[k]
    text = cases.run_engine(_case([read]), dict(), dump=False).text
    assert _block(text) == want


@pytest.mark.gpu
@pytest.mark.parametrize("d", sorted(D_TABLE))
def test_engine_max_count_table(d):
    text = cases.run_engine(_d_case(), dict(max_cnt=d), dump=False).text
    assert [int(l.split("\t")[3]) for l in text.strip().split("\n")] == D_TABLE[d]


# ---- BASELINE config 2b: test-data/twolib.sorted.cram (-p, -l twolib_site_list.txt, -f rand1k.fa) -------------------------
# CRAM decode is host I/O outside the hot path; the fixture's four records (samtools view: 60M, MAPQ 60, no qualities -> 0xFF,
# NM:i:0, RG reads{1,2}_id -> LB reads{1,2}_lb, starts 1/61/121/181) are rebuilt here and the output is compared with what the
# reference binary prints for the CRAM itself (tests/golden/ref_cram_twolib_*.txt.gz, made by make_golden.py).
def _cram_case():
    import os
    from bam_readcount_b200.bamio import Fasta
    fa = Fasta(os.path.join(cases.GOLDEN, "rand1k.fa"))
    ref = fa.fetch("rand1k")
    bb = BatchBuilder()
    for i, (start, lib) in enumerate(((0, 0), (60, 0), (120, 1), (180, 1))):
        bb.add_sam(tid=0, pos=start, flag=0, mapq=60, lib=lib, cigar="60M", seq=ref[start:start + 60].decode(),
                   qual=np.full(60, 255, np.uint8), nm=0, sm=None, qname=f"read{lib + 1}-{i % 2 + 1}")
    return dict(name="cram", contigs=[("rand1k", 1000, ref, 0)], batch=bb.build(), regions=[(0, 50, 60)], site_list=True,
                lib_names=["reads1_lb", "reads2_lb"])


@pytest.mark.parametrize("per_lib", [True, False])
def test_oracle_cram_fixture_records(per_lib):
    text, _, _ = cases.run_oracle(_cram_case(), dict(per_lib=per_lib))
    want = cases.load_golden_text("ref_cram_twolib_perlib.txt" if per_lib else "ref_cram_twolib_alllib.txt")
    assert text == want and len(want.splitlines()) == 11
    assert "A:1:60.00:255.00:60.00:1:0:0.37:0.00:0.00:1:0.15:60.00:0.15" in want.splitlines()[0]   # SURVEY.md Appendix E


@pytest.mark.gpu
@pytest.mark.parametrize("per_lib", [True, False])
def test_engine_cram_fixture_records(per_lib):
    text = cases.run_engine(_cram_case(), dict(per_lib=per_lib), dump=False).text
    assert text == cases.load_golden_text("ref_cram_twolib_perlib.txt" if per_lib else "ref_cram_twolib_alllib.txt")
