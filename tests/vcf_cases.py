"""Inputs of the --vcf tests: VCF text over the reference's test.bam fixture, its sample-column variants, and a BGZF writer."""
from __future__ import annotations

import bam_craft
import cases

HEAD = "##fileformat=VCFv4.2\n##contig=<ID=21>\n##FORMAT=<ID=GT,Number=1,Type=String,Description=\"Genotype\">\n"


def fixture_records():
    """Records around the fixture's two covered sites: SNVs (all four bases, multi-allelic), insertions, deletions of several
    lengths, MNPs, '*', '<DEL>', lower case, a REF with an IUPAC letter, an N reference, a contig the BAM lacks and
    uncovered positions.  Each is (CHROM, POS, REF, ALT)."""
    chr21 = cases.testbam_chr21()
    ref = lambda p, n=1: chr21[p - 1:p - 1 + n].decode("latin-1").upper()        # 1-based
    out = []
    for site in (10402985, 10405200):
        for p in range(site - 6, site + 7):
            r = ref(p)
            alts = [b for b in "ACGT" if b != r]
            out.append(("21", p, r, ",".join(alts)))
            out.append(("21", p, r, r + "A," + r + "CT"))
            out.append(("21", p, ref(p, 2), r))
            out.append(("21", p, ref(p, 3), r + "," + ref(p + 1, 2)[::-1]))
        out.append(("21", site, ref(site).lower(), "a,<DEL>,*," + ref(site).lower() + "g"))
        out.append(("21", site + 1, ref(site + 1, 2), "TT,.,A"))
        out.append(("21", site, "N", "A,C"))
        out.append(("21", site, "R", "A"))
    out += [("chrZ", 100, "A", "C"), ("21", 10300000, "A", "G,AT"), ("21", 10300000, "AC", "A"), ("21", 1, "A", "G")]
    return out


def vcf_text(records, samples=("S1",), sites_only=False, pad=False) -> str:
    """A VCF of the records.  Sample columns hold a GT (the chosen sample's '.' when pad, so its values are padded)."""
    out = HEAD
    cols = "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO"
    out += cols + ("" if sites_only else "\tFORMAT\t" + "\t".join(samples)) + "\n"
    for k, (c, p, r, a) in enumerate(records):
        line = f"{c}\t{p}\trec{k}\t{r}\t{a}\t50\tPASS\tDP=10"
        if not sites_only:
            line += "\tGT:GQ\t" + "\t".join("." if pad and i == 0 else f"0/1:{k % 50}" for i in range(len(samples)))
        out += line + "\n"
    return out


def write_bgzf(path: str, data: bytes):
    """bgzip's format: BGZF members of at most 64 KiB and the empty end-of-file member."""
    with open(path, "wb") as fh:
        for i in range(0, len(data), 0xff00):
            fh.write(bam_craft.bgzf_member(data[i:i + 0xff00]))
        fh.write(bam_craft.bgzf_member(b""))


write_fasta21 = cases.write_testbam_fasta        # the name tests/golden/make_vcf_golden.py writes the fixture's ref.fa with
