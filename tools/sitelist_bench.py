"""Site-list mode (-l) wall-clock: brc-readcount vs the reference binary on the same synthetic BAM and the same list of
single-base sites.  usage: sitelist_bench.py [contig_len] [site_step] [ref_sites]"""
import os, subprocess, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bam_readcount_b200 import synth, build
from oracle.oracle import REF_BIN, REF_SAMTOOLS
L = int(float(sys.argv[1])) if len(sys.argv) > 1 else 2_000_000
step = int(sys.argv[2]) if len(sys.argv) > 2 else 20
ref_sites = int(sys.argv[3]) if len(sys.argv) > 3 else 2000
d = tempfile.mkdtemp()
ref = synth.synth_reference(L, 1234); b = synth.synth_reads(ref, 30, seed=1234)
synth.write_fasta(d + "/ref.fa", "chr1", ref)
synth.write_sam(d + "/s.sam", b, [("chr1", L)])
subprocess.check_call([REF_SAMTOOLS, "view", "-b", "-o", d + "/s.bam", d + "/s.sam"]); subprocess.check_call([REF_SAMTOOLS, "index", d + "/s.bam"])
sites = list(range(1000, L - 1000, step))
with open(d + "/sites", "w") as fh:
    fh.write("".join(f"chr1\t{p}\t{p}\n" for p in sites))
with open(d + "/sites_ref", "w") as fh:
    fh.write("".join(f"chr1\t{p}\t{p}\n" for p in sites[:ref_sites]))
print(f"BAM: {b.n_reads} reads; {len(sites)} sites every {step} bp")
exe = build.build_cli()
t0 = time.time()
with open(d + "/out.txt", "wb") as fh:
    p = subprocess.run([exe, "-w", "0", "-q", "20", "-b", "20", "-f", d + "/ref.fa", "-l", d + "/sites", d + "/s.bam"], stdout=fh, stderr=subprocess.PIPE,
                       env=dict(os.environ, BRC_CLI_TIMING="1"))
dt = time.time() - t0
out = open(d + "/out.txt", "rb").read()
print(f"brc-readcount: {dt:.2f}s  {len(sites)/dt:.3e} sites/s rc={p.returncode}\n   " + "\n   ".join(p.stderr.decode().strip().splitlines()[-2:]))
t0 = time.time()
r = subprocess.run([REF_BIN, "-w", "0", "-q", "20", "-b", "20", "-f", d + "/ref.fa", "-l", d + "/sites_ref", d + "/s.bam"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
dt = time.time() - t0
print(f"reference binary on the first {ref_sites} sites: {dt:.2f}s  {ref_sites/dt:.3e} sites/s")
print("byte-identical on those sites:", out.startswith(r.stdout))
