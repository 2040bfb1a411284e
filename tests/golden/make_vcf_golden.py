"""Writes vcf_sha256.json: SHA-256 of the reference binary's STDOUT over the site list the --vcf fixture derives
(tests/vcf_cases.py) from the reference's test.bam, per flag set.  Run where oracle/_ref/bam-readcount exists."""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]
import vcf_cases  # noqa: E402
import vcf_rule  # noqa: E402

REF_BIN = os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref", "bam-readcount")
FLAGS = {"fixture_default": [], "fixture_ic": ["-i"], "fixture_q20b20": ["-q", "20", "-b", "20"]}

if __name__ == "__main__":
    out = {}
    with tempfile.TemporaryDirectory() as d:
        fa = vcf_cases.write_fasta21(os.path.join(d, "ref.fa"))
        sl = os.path.join(d, "sites")
        open(sl, "w").write(vcf_rule.derive(vcf_cases.vcf_text(vcf_cases.fixture_records())))
        for key, flags in FLAGS.items():
            p = subprocess.run([REF_BIN] + flags + ["-w", "0", "-f", fa, "-l", sl, os.path.join(HERE, "test.bam")], capture_output=True, check=True)
            out[key] = hashlib.sha256(p.stdout).hexdigest()
    with open(os.path.join(HERE, "vcf_sha256.json"), "w") as fh:
        json.dump(out, fh, indent=1, sort_keys=True)
        fh.write("\n")
