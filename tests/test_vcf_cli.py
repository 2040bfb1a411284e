"""CPU: the --vcf contract without a device.  The allele rule on hand-written lines (tests/vcf_rule.py, the GPU tests' oracle),
every refusal of `brc-readcount --vcf` (exit 1, a message, nothing on STDOUT), and the site list it derives: under
BRC_CLI_DECODE_ONLY=1 a --vcf run prints the decode summary of exactly the regions `-l <derived site list>` fetches."""
import os
import subprocess

import pytest

import cases
import vcf_cases
import vcf_rule
from cases import DECODE_ONLY

BAM = os.path.join(cases.GOLDEN, "test.bam")


def _line(chrom, pos, ref, depth, entries):
    """A readcount line: entries {name: (count, plus, minus)}; the six base entries are always printed."""
    zero = "0:0.00:0.00:0.00:0:0:0.00:0.00:0.00:0:0.00:0.00:0.00"
    out = f"{chrom}\t{pos}\t{ref}\t{depth}"
    for b in "=ACGTN":
        c = entries.get(b)
        out += f"\t{b}:" + (zero if c is None else f"{c[0]}:60.00:30.00:0.00:{c[1]}:{c[2]}:0.50:0.00:0.00:0:0.00:100.00:0.50")
    for k, c in entries.items():
        if k[0] in "+-":
            out += f"\t{k}:{c[0]}:60.00:0.00:0.00:{c[1]}:{c[2]}:0.50:0.00:0.00:0:0.00:100.00:0.50"
    return out + "\n"


def _vcf(rows, samples=("S1",), sites_only=False, pad=False):
    return vcf_cases.vcf_text(rows, samples=samples, sites_only=sites_only, pad=pad)


def _record_values(annotated: str):
    """The last column of every data line."""
    return [ln.split("\t")[-1] for ln in annotated.splitlines() if ln and not ln.startswith("#")]


def test_rule_each_allele_shape():
    text = (_line("21", 100, "A", 20, {"A": (12, 7, 5), "G": (5, 2, 3), "+CT": (2, 1, 1)}) +
            _line("21", 201, "C", 9, {"C": (6, 3, 3), "-CG": (3, 2, 1), "-C": (1, 0, 1)}))
    vcf = _vcf([("21", 100, "A", "G"), ("21", 100, "a", "act,aG"), ("21", 200, "TC", "T"), ("21", 200, "TCG", "t"),
                ("21", 200, "TCGA", "T")])
    got = _record_values(vcf_rule.annotate(vcf, text))
    assert got == ["0/1:0:20:12,5:7,2:5,3:0.25",
                   "0/1:1:20:12,2,0:7,1,0:5,1,0:0.1,0",        # +CT present; +G absent (0)
                   "0/1:2:9:6,1:3,0:3,1:0.111111",            # a one-base deletion: the line after the anchor
                   "0/1:3:9:6,3:3,2:3,1:0.333333",
                   "0/1:4:9:6,0:3,0:3,0:0"]


def test_rule_uncountable_alts_missing_line_and_contig():
    text = _line("21", 100, "A", 3, {"A": (3, 3, 0)})
    vcf = _vcf([("21", 100, "A", "GT,*,<DEL>,.,C"), ("21", 100, "AC", "GT"), ("21", 100, "R", "A"), ("21", 50, "A", "C"),
                ("chrZ", 100, "A", "C"), ("21", 100, "N", "A")])
    got = _record_values(vcf_rule.annotate(vcf, text, contigs=["21"]))
    assert got == ["0/1:0:3:3,.,.,.,.,0:3,.,.,.,.,0:0,.,.,.,.,0:.,.,.,.,0",
                   "0/1:1:.:.:.:.:.",                           # MNP only: not counted
                   "0/1:2:.:.:.:.:.",                           # IUPAC REF: nothing countable
                   "0/1:3:0:0,0:0,0:0,0:.",                     # counted, no line: DP 0, AF '.'
                   "0/1:4:.:.:.:.:.",                           # contig missing from the BAM
                   "0/1:5:3:0,3:0,3:0,0:1"]                     # N reference: the REF entry is N's
    assert vcf_rule.derive(vcf) == "21\t100\t100\n21\t50\t50\nchrZ\t100\t100\n21\t100\t100\n"


def test_rule_derive_and_format_fields():
    vcf = _vcf([("21", 100, "A", "G"), ("21", 100, "AC", "A"), ("21", 7, "AC", "GT"), ("chrZ", 5, "A", "T")])
    assert vcf_rule.derive(vcf) == "21\t100\t100\n21\t101\t101\nchrZ\t5\t5\n"
    out = vcf_rule.annotate(vcf, _line("21", 100, "A", 7, {"A": (4, 2, 2), "G": (3, 1, 2)}))
    lines = out.splitlines()
    i = [k for k, ln in enumerate(lines) if ln.startswith("#CHROM")][0]
    assert lines[i - 5:i] == vcf_rule.HEADER.splitlines()
    assert lines[i + 1].split("\t")[8] == "GT:GQ:BRC_DP:BRC_AD:BRC_ADF:BRC_ADR:BRC_AF"
    assert lines[i + 1].split("\t")[9] == "0/1:0:7:4,3:2,1:2,2:0.428571"      # %.6g


def test_rule_padding_sites_only_and_sample_choice():
    text = _line("21", 100, "A", 4, {"A": (4, 4, 0)})
    rows = [("21", 100, "A", "C")]
    padded = vcf_rule.annotate(_vcf(rows, pad=True), text)
    assert padded.splitlines()[-1].split("\t")[9] == ".:.:4:4,0:4,0:0,0:0"
    so = vcf_rule.annotate(_vcf(rows, sites_only=True), text, sample="NEW")
    assert [ln for ln in so.splitlines() if ln.startswith("#CHROM")][0].endswith("\tINFO\tFORMAT\tNEW")
    assert so.splitlines()[-1].split("\t")[8:] == ["BRC_DP:BRC_AD:BRC_ADF:BRC_ADR:BRC_AF", "4:4,0:4,0:0,0:0"]
    multi = vcf_rule.annotate(_vcf(rows, samples=("S1", "S2", "S3")), text, sample="S2")
    c = multi.splitlines()[-1].split("\t")
    assert c[9] == "0/1:0" and c[10] == "0/1:0:4:4,0:4,0:0,0:0" and c[11] == "0/1:0"


def _run(args, vcf_path, env=DECODE_ONLY):
    return subprocess.run([cases.cli()] + args + ["--vcf", vcf_path, BAM], capture_output=True, env=env)


def test_cli_vcf_refusals(tmp_path):
    exe = cases.cli()
    good = tmp_path / "good.vcf"
    good.write_text(_vcf([("21", 10402985, "A", "C")]))
    multi = tmp_path / "multi.vcf"
    multi.write_text(_vcf([("21", 10402985, "A", "C")], samples=("S1", "S2", "S1")))
    so = tmp_path / "so.vcf"
    so.write_text(_vcf([("21", 10402985, "A", "C")], sites_only=True))
    bad = {
        "short": (vcf_cases.HEAD + "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tS1\n21\t5\t.\tA\tC\n", b"line 5: fewer than 8 columns"),
        "pos": (_vcf([("21", 0, "A", "C")]), b"line 5: POS is not a positive integer"),
        "pos2": (_vcf([("21", "12x", "A", "C")]), b"line 5: POS is not a positive integer"),
        "early": ("##fileformat=VCFv4.2\n21\t5\t.\tA\tC\t.\t.\t.\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\n", b"line 2: data before the #CHROM"),
        "cols": (_vcf([("21", 5, "A", "C")]).rstrip("\n") + "\textra\n", b"line 5: 11 columns, the #CHROM line has 10"),
        "brc": ("##FORMAT=<ID=BRC_AD,Number=R,Type=Integer,Description=\"x\">\n" + _vcf([("21", 5, "A", "C")]), b"already declares a BRC_* FORMAT"),
        "nochrom": ("##fileformat=VCFv4.2\n", b"no #CHROM header line"),
    }
    for name, (text, msg) in bad.items():
        f = tmp_path / f"{name}.vcf"
        f.write_text(text)
        p = _run([], str(f))
        assert p.returncode == 1 and msg in p.stderr and p.stdout == b"", (name, p.stderr)
    gz = tmp_path / "plain.vcf.gz"
    import gzip
    gz.write_bytes(gzip.compress(good.read_bytes()))
    p = _run([], str(gz))
    assert p.returncode == 1 and b"not BGZF" in p.stderr and p.stdout == b""
    for args, path, msg in ((["--vcf-sample", "X"], good, b"--vcf-sample X: no such sample"),
                            ([], multi, b"--vcf-sample NAME is required"),
                            (["--vcf-sample", "S1"], multi, b"is ambiguous: 2 sample columns"),
                            ([], so, b"--vcf-sample NAME names the one added"),
                            ([], tmp_path / "missing.vcf", b"cannot open")):
        p = _run(args, str(path))
        assert p.returncode == 1 and msg in p.stderr and p.stdout == b"", (args, p.stderr)
    lst = tmp_path / "list"
    lst.write_text(f"{BAM}\t{tmp_path / 'o'}\n")
    for extra, what in ((["-l", str(good)], b"-l"), (["-p"], b"-p"), (["--min-alt-count", "2"], b"--min-alt-count"),
                        (["--min-alt-fraction", "0.1"], b"--min-alt-count/--min-alt-fraction"), (["--shard", "0/2"], b"--shard")):
        p = _run(extra, str(good))
        assert p.returncode == 1 and b"--vcf cannot be combined with " + what in p.stderr and p.stdout == b"", (extra, p.stderr)
    p = subprocess.run([exe, "--vcf", str(good), BAM, "21:1-100"], capture_output=True, env=DECODE_ONLY)
    assert p.returncode == 1 and b"cannot be combined with positional regions" in p.stderr and p.stdout == b""
    p = subprocess.run([exe, "--vcf", str(good), "--bam-list", str(lst)], capture_output=True, env=DECODE_ONLY)
    assert p.returncode == 1 and b"cannot be combined with --bam-list" in p.stderr and p.stdout == b""
    assert not os.path.exists(tmp_path / "o")
    p = subprocess.run([exe, "--vcf-sample", "S1", BAM, "21:1-100"], capture_output=True, env=DECODE_ONLY)
    assert p.returncode == 1 and b"--vcf-sample needs --vcf" in p.stderr and p.stdout == b""


@pytest.mark.parametrize("form", ["plain", "bgzf"])
@pytest.mark.parametrize("shape", ["one", "multi", "sites_only"])
def test_cli_vcf_derivation_equals_derived_site_list(tmp_path, form, shape):
    """--vcf fetches exactly the regions of `-l derived`: same decode summary on STDOUT, same STDERR (the 'not found' lines)."""
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
    sl.write_text(vcf_rule.derive(text))
    want = subprocess.run([exe, "-l", str(sl), BAM], capture_output=True, env=DECODE_ONLY)
    extra = [] if shape == "one" else ["--vcf-sample", "S2" if shape == "multi" else "NEW"]
    got = subprocess.run([exe, "--vcf", str(path)] + extra + [BAM], capture_output=True, env=DECODE_ONLY)
    assert want.returncode == 0 and got.returncode == 0, got.stderr.decode()
    assert got.stdout == want.stdout and len(want.stdout.splitlines()) == len(sl.read_text().splitlines()) - sl.read_text().count("chrZ")
    assert got.stderr == want.stderr and b"chrZ not found in bam file. Region chrZ 100 100 skipped." in got.stderr


def test_allele_query_symbols_exported():
    from bam_readcount_b200 import engine
    lib = engine.load_library()
    assert hasattr(lib, "brc_set_allele_queries") and hasattr(lib, "brc_get_allele_answers")
    assert lib.brc_abi_version() == 2
    assert engine.ALLELE_ANSWER.itemsize == 64


@pytest.mark.parametrize("key,flags", [("fixture_default", {}), ("fixture_ic", dict(insertion_centric=True)),
                                       ("fixture_q20b20", dict(min_mapq=20, min_bq=20))])
def test_oracle_text_over_derived_sites_is_the_reference_binarys(key, flags):
    """The C oracle's text over the fixture's derived site list hashes to what the reference binary printed
    (tests/golden/vcf_sha256.json, make_vcf_golden.py): the text the GPU tests annotate is pinned to the reference."""
    case = cases.testbam_case()
    sites = [ln.split("\t") for ln in vcf_rule.derive(vcf_cases.vcf_text(vcf_cases.fixture_records())).splitlines()]
    case = dict(case, regions=[(0, int(b), int(e)) for c, b, e in sites if c == "21"])
    cases.assert_anchor("vcf_sha256.json", key, cases.run_oracle(case, flags).text)
