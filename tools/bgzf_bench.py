"""BGZF output compressed on the device (brc_bgzf_*, `brc-readcount --bgzf`): throughput, ratio and CLI wall time.

Device: the golden readcount texts, repeated to --mb MB, through a BgzfWriter into /dev/null: the chunks' kernels alone (CUDA
events, brc_bgzf_stats) and the writer end to end from host buffers, in GB/s of input; the ratio against zlib levels 1 and 6 on
the same 65280-byte blocks.  CLI: brc-readcount on a synthetic BAM of --cli-mb Mb with -i (DESIGN.md §10's), plain into
/dev/null, --bgzf into /dev/null, plain | gzip -1 (when gzip exists) and plain into a multi-threaded Python zlib writer.  Median
of --runs runs each.  Prints one JSON object with the card's name and power limit read in the same call."""
import argparse
import concurrent.futures
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
BLOCK = 0xff00


def card():
    q = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
    name, pl = [x.strip() for x in q.strip().split(",")]
    return name, pl


def zlib_blocks(data, level):
    return sum(len(zlib.compress(data[i:i + BLOCK], level)) - 6 + 26 for i in range(0, len(data), BLOCK)) + 28


def device(args):
    import cases
    from bam_readcount_b200.engine import BgzfWriter
    g = os.path.join(ROOT, "tests", "golden")
    text = b"".join(cases.load_golden_text(f[:-3]).encode("latin-1") for f in sorted(os.listdir(g)) if f.endswith(".txt.gz"))
    data = (text * (int(args.mb * 1e6) // len(text) + 1))[:int(args.mb * 1e6)]
    fd = os.open("/dev/null", os.O_WRONLY)
    mv = memoryview(data)
    walls, kernels, out_bytes = [], [], 0
    for r in range(args.runs + 1):                       # the first run warms up the context and the allocations
        t0 = time.perf_counter()
        w = BgzfWriter(fd)
        for i in range(0, len(data), 4 << 20):           # 4 MB writes, as a formatter hands over its parts
            w.write(mv[i:i + (4 << 20)])
        st = w.stats()
        w.close()
        dt = time.perf_counter() - t0
        if r:
            walls.append(dt); kernels.append(st["kernel_ms"]); out_bytes = st["bytes_out"]
    os.close(fd)
    sample = data[:min(len(data), 64 << 20)]
    return {"input_MB": len(data) / 1e6, "output_MB": out_bytes / 1e6, "ratio": len(data) / max(out_bytes, 1),
            "kernels_GBps": len(data) / 1e9 / (statistics.median(kernels) / 1e3),
            "writer_end_to_end_GBps": len(data) / 1e9 / statistics.median(walls),
            "zlib1_ratio": len(sample) / zlib_blocks(sample, 1), "zlib6_ratio": len(sample) / zlib_blocks(sample, 6),
            "zlib_sample_MB": len(sample) / 1e6}


def threaded_zlib_sink(src, workers):
    """Reads src to its end, compressing 65280-byte blocks at level 1 on `workers` threads (zlib releases the GIL)."""
    out = 0
    with concurrent.futures.ThreadPoolExecutor(workers) as ex:
        pend = []
        while True:
            buf = src.read(BLOCK * 64)
            if not buf:
                break
            pend.append(ex.submit(lambda b: sum(len(zlib.compress(b[i:i + BLOCK], 1)) for i in range(0, len(b), BLOCK)), buf))
            if len(pend) > 2 * workers:
                out += pend.pop(0).result()
        out += sum(p.result() for p in pend)
    return out


def cli(args):
    from bam_readcount_b200 import build, synth_cb
    from oracle.oracle import REF_SAMTOOLS
    exe = build.build_cli()
    nblk = int(args.cli_mb * 1e6) // synth_cb.BLOCK_BP
    spec = synth_cb.Spec(seed=77, mode=synth_cb.WGS, n_libs=8, contig_len=(nblk + 4) * synth_cb.BLOCK_BP)
    res = {}
    with tempfile.TemporaryDirectory() as wd:
        info = synth_cb.write_sample_bam(spec, 0, 0, nblk, wd, REF_SAMTOOLS)
        base = [exe, "-w", "0", "-i", "-f", info["fasta"], info["bam"], f"chr1:1001-{nblk * synth_cb.BLOCK_BP}"]
        ways = {"plain": None, "bgzf": None, "python_zlib_threads": None}
        if shutil.which("gzip"):
            ways["gzip_1"] = None
        times = {k: [] for k in ways}
        for r in range(args.runs + 1):
            for k in ways:
                t0 = time.perf_counter()
                if k == "plain":
                    with open(os.devnull, "wb") as fh:
                        rc = subprocess.run(base, stdout=fh, stderr=subprocess.DEVNULL).returncode
                elif k == "bgzf":
                    with open(os.devnull, "wb") as fh:
                        rc = subprocess.run(base[:1] + ["--bgzf"] + base[1:], stdout=fh, stderr=subprocess.DEVNULL).returncode
                elif k == "gzip_1":
                    with open(os.devnull, "wb") as fh:
                        rc = subprocess.run(" ".join(base) + " 2>/dev/null | gzip -1", shell=True, stdout=fh).returncode
                else:
                    p = subprocess.Popen(base, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
                    threaded_zlib_sink(p.stdout, os.cpu_count() or 4)
                    rc = p.wait()
                dt = time.perf_counter() - t0
                assert rc == 0, k
                if r:
                    times[k].append(dt)
        res = {k + "_s": statistics.median(v) for k, v in times.items()}
        res["bgzf_over_plain"] = res["bgzf_s"] / res["plain_s"]
        res["cli_region_Mb"] = nblk * synth_cb.BLOCK_BP / 1e6
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=float, default=1024)
    ap.add_argument("--cli-mb", type=float, default=4)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--no-cli", action="store_true")
    args = ap.parse_args()
    name, pl = card()
    out = {"gpu": name, "power_limit": pl, "runs": args.runs, "host_cpus": os.cpu_count()}
    out.update(device(args))
    if not args.no_cli:
        out.update(cli(args))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
