"""CPU: the --vcf-complex contract without a device.  The complex rule (tests/complex_rule.py, the GPU tests' oracle) on a
hand-built BAM; the kernel's flank walk (brc_complex.cuh, compiled with g++) against the rule's on every read of three BAMs;
and, under BRC_CLI_DECODE_ONLY=1, the site list --vcf --vcf-complex derives and every refusal."""
import os
import subprocess

import numpy as np
import pytest

import cases
import complex_cases
import complex_rule
import vcf_cases
from bam_readcount_b200 import bamio
from bam_readcount_b200.engine import admitted
from cases import DECODE_ONLY

BAM = os.path.join(cases.GOLDEN, "test.bam")


def _crafted_batch(tmp_path):
    bam, _ = complex_cases.write_crafted(str(tmp_path))
    return bamio.read_bam(bam)[1]


def test_rule_on_crafted_reads(tmp_path):
    batch = _crafted_batch(tmp_path)
    rows = complex_cases.crafted_reads()
    P = complex_cases.P
    reads = complex_rule.Reads(batch)
    # every read's allele string, as the crafted alignment says it is
    for k, (name, pos, _, seq, _, flag, _, want) in enumerate(rows):
        c0, c1 = int(batch.cigar_off[k]), int(batch.cigar_off[k + 1])
        f = complex_rule.resolve(batch.cigar[c0:c1].tolist(), pos, P - 1, P + 2)
        got = None if f is None or flag & complex_rule.FLAG_FILTER else seq[f[0] + 1:f[1]].replace("R", "N")
        assert got == want, name
    al = list(complex_cases.crafted_alleles())
    by = {r[0]: r for r in rows}

    def expect(names):
        s = [by[n][7] for n in names if by[n][7] is not None]
        plus = [by[n][7] for n in names if by[n][7] is not None and not by[n][5] & 16]
        return len(s), [(s.count(a), plus.count(a), s.count(a) - plus.count(a)) for a in al]
    everything = [r[0] for r in rows]
    dp, got = complex_rule.count(reads, P, 2, al)
    assert (dp, got) == expect(everything) and dp == 13 and got[1] == (5, 4, 1)
    # -q 20 -b 20: the low-MAPQ read and the read with a low base inside S go; the one with a low base outside stays
    q = complex_rule.count(reads, P, 2, al, min_mapq=20, min_bq=20)
    assert q == expect([n for n in everything if n not in ("low_mapq", "low_quality_inside")])
    # -d 3: the pileup buffer keeps three of the reads starting at 80
    kept = admitted(batch, 0, 3)
    assert len(kept) < batch.n_reads
    assert complex_rule.count(complex_rule.Reads(batch, kept), P, 2, al) == expect([rows[i][0] for i in kept])
    # a right flank past the contig: zero counts
    assert complex_rule.count(reads, complex_cases.L - 2, 2, ["AC"], chrom_len=complex_cases.L) == (0, [(0, 0, 0)])


def test_rule_classifies_and_derives():
    assert complex_rule.complex_alleles(5, "CC", ["TT"]) == ("CC", ["TT"])
    assert complex_rule.complex_alleles(5, "atg", ["c", "<DEL>"]) == ("ATG", ["C", None])
    assert complex_rule.complex_alleles(5, "A", ["T", "GC"]) == ("A", ["T", "GC"])             # mixed: the whole record
    assert complex_rule.complex_alleles(1, "CC", ["TT"]) is None                              # POS 1: no left flank
    for ref, alts in (("A", ["T", "AC"]), ("AC", ["A"]), ("CC", ["*", "<INV>", "."]), ("CR", ["TT"])):
        assert complex_rule.complex_alleles(5, ref, alts) is None, (ref, alts)
    text = vcf_cases.vcf_text([("21", 10, "CC", "TT"), ("21", 20, "AC", "A"), ("21", 30, "A", "T,GC"), ("21", 1, "CC", "TT")])
    assert complex_rule.derive(text) == "21\t10\t10\n21\t21\t21\n21\t30\t30\n"
    assert complex_rule.complex_values(4, [(1, 1, 0), (2, 0, 2)], ["TT", None]) == "4:1,2,.:1,0,.:0,2,.:0.5,."


def test_device_resolver_equals_rule(tmp_path):
    """The kernel's flank walk, compiled for the CPU, gives the rule's flank query positions (or 'does not span') for every read
    of test.bam, the crafted BAM and a synthetic BAM over spans of lengths 1-20 placed all along each read."""
    from bam_readcount_b200 import synth
    exe = cases.check_program("complex_check")
    ref = synth.synth_reference(4000, 5)
    batches = [cases.testbam_case()["batch"], _crafted_batch(tmp_path), synth.synth_reads(ref, 20, seed=5)]
    rng = np.random.default_rng(3)
    lines, want = [], []
    for b in batches:
        end = b.ref_end()
        for i in range(b.n_reads):
            cig = b.cigar[int(b.cigar_off[i]):int(b.cigar_off[i + 1])].tolist()
            p, e = int(b.pos[i]), int(end[i])
            for left in sorted(set(rng.integers(p - 3, e + 2, 14).tolist()) | {p - 1, p, e - 2, e - 1}):
                n = int(rng.integers(1, 21))
                lines.append(f"{p} {left} {left + n + 1} {len(cig)} " + " ".join(map(str, cig)))
                f = complex_rule.resolve(cig, p, left, left + n + 1)
                want.append("-1 -1" if f is None else f"{f[0]} {f[1]}")
    out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout.splitlines()
    assert len(out) == len(want) > 10000
    bad = [(lines[k], out[k], want[k]) for k in range(len(want)) if out[k] != want[k]]
    assert not bad, bad[:5]
    assert sum(w != "-1 -1" for w in want) > len(want) // 4


@pytest.mark.parametrize("form", ["plain", "bgzf"])
@pytest.mark.parametrize("shape", ["one", "multi", "sites_only"])
def test_derivation_equals_derived_site_list(tmp_path, form, shape):
    """--vcf --vcf-complex fetches exactly the regions of `-l complex_rule.derive`: same decode summary, same STDERR."""
    exe = cases.cli()
    recs = vcf_cases.fixture_records()
    text = vcf_cases.vcf_text(recs, samples=("S1", "S2") if shape == "multi" else ("S1",), sites_only=shape == "sites_only")
    path = tmp_path / "in.vcf"
    if form == "plain":
        path.write_text(text)
    else:
        path = tmp_path / "in.vcf.gz"
        vcf_cases.write_bgzf(str(path), text.encode())
    sl = tmp_path / "derived"
    sl.write_text(complex_rule.derive(text))
    import vcf_rule
    assert len(complex_rule.derive(text).splitlines()) > len(vcf_rule.derive(text).splitlines())   # the fixture has complex records
    want = subprocess.run([exe, "-l", str(sl), BAM], capture_output=True, env=DECODE_ONLY)
    extra = [] if shape == "one" else ["--vcf-sample", "S2" if shape == "multi" else "NEW"]
    got = subprocess.run([exe, "--vcf", str(path), "--vcf-complex"] + extra + [BAM], capture_output=True, env=DECODE_ONLY)
    assert want.returncode == 0 and got.returncode == 0, got.stderr.decode()
    assert got.stdout == want.stdout and got.stderr == want.stderr


def test_refusals(tmp_path):
    exe = cases.cli()
    good = tmp_path / "good.vcf"
    good.write_text(vcf_cases.vcf_text([("21", 10402985, "AC", "TT")]))
    p = subprocess.run([exe, "--vcf-complex", BAM, "21:1-100"], capture_output=True, env=DECODE_ONLY)
    assert p.returncode == 1 and b"--vcf-complex needs --vcf" in p.stderr and p.stdout == b""
    lst = tmp_path / "list"
    lst.write_text(f"{BAM}\t{tmp_path / 'o'}\n")
    for extra, what in ((["-l", str(good)], b"-l"), (["-p"], b"-p"), (["--min-alt-count", "2"], b"--min-alt-count"),
                        (["--shard", "0/2"], b"--shard"), (["--bam-list", str(lst)], b"--bam-list")):
        args = [exe, "--vcf", str(good), "--vcf-complex"] + extra + ([] if "--bam-list" in extra else [BAM])
        p = subprocess.run(args, capture_output=True, env=DECODE_ONLY)
        assert p.returncode == 1 and b"--vcf cannot be combined with " + what in p.stderr and p.stdout == b"", (extra, p.stderr)
    p = subprocess.run([exe, "--vcf", str(good), "--vcf-complex", BAM, "21:1-100"], capture_output=True, env=DECODE_ONLY)
    assert p.returncode == 1 and b"cannot be combined with positional regions" in p.stderr and p.stdout == b""
    bad = tmp_path / "bad.vcf"
    bad.write_text(vcf_cases.vcf_text([("21", 0, "AC", "TT")]))
    p = subprocess.run([exe, "--vcf", str(bad), "--vcf-complex", BAM], capture_output=True, env=DECODE_ONLY)
    assert p.returncode == 1 and b"POS is not a positive integer" in p.stderr and p.stdout == b""
    assert not os.path.exists(tmp_path / "o")
    p = subprocess.run([exe], capture_output=True)
    assert b"--vcf-complex" in p.stderr + p.stdout


def test_complex_symbols_exported():
    from bam_readcount_b200 import engine
    lib = engine.load_library()
    assert hasattr(lib, "brc_set_complex_queries") and hasattr(lib, "brc_get_complex_answers")
    assert engine.COMPLEX_COUNT.itemsize == 8
    assert engine.C.sizeof(engine.CComplexQuery) == 24 and engine.C.sizeof(engine.CComplexAllele) == 16
