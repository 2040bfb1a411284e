"""Speed of the counter-based read generator (csrc/brc_synth.cu) on the GPU; prints one JSON line.

Two shapes: one full C4 window (blocks 0-9766 of contig 0: 2.5 M reads) and one C5 launch (296 sites x 50 000 reads).
For each: the whole fill (count, scan and fill kernels) timed with CUDA events, median of --runs after --warmup, and each
kernel's own time from torch.profiler (mean over --runs, in a run of its own).  The bytes a fill writes over its time gives
its achieved write bandwidth.

--lib PATH (repeatable) times other builds of libbrc_synth.so in the same process, runs alternating, and checks that every
build writes the same bytes as the first.  --bench also runs bench.py (C4, resident windows, then --no-resident): the gap
between the two is what regenerating windows costs once it overlaps the engine's streams.

    python tools/synth_bench.py [--runs 20] [--warmup 3] [--lib other/libbrc_synth.so] [--bench]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KERNELS = ("synth_count_kernel", "synth_scan_kernel", "synth_fill_kernel")


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], text=True).strip()
    except Exception:
        pl = None
    return name, pl


def shapes():
    from bam_readcount_b200 import synth_cb as sc
    c4 = sc.Spec(seed=1234, mode=sc.WGS, n_libs=8, contig_len=97656 * sc.BLOCK_BP, n_contigs=24)
    c5 = sc.Spec(seed=1234, mode=sc.DEEP, n_libs=8, depth=50_000, site_stride=1000, n_sites=10_000, contig_len=sc.BLOCK_BP)
    return {"c4_window": (c4, 0, 0, -(-97656 // 10)), "c5_launch": (c5, 0, 0, 296)}


def fill_fn(lib, dw, contig, lo, hi, stream_ptr):
    """DeviceWindow.fill through a given build of the library."""
    from bam_readcount_b200 import synth_cb as sc
    t = dw.t
    n = dw.spec.window_reads(lo, hi)
    out = sc.COut(n, None, *[t[k].data_ptr() for k in ("pos", "flag", "mapq", "lib", "l_qseq", "nm", "sm", "cigar_off", "cigar", "seq_off",
                                                       "seq", "qual_off", "qual")], t["region"].data_ptr())
    spec_c = dw.spec.c

    def go():
        rc = lib.brc_synth_fill_device(C.byref(spec_c), contig, lo, hi, C.byref(out), t["scratch"].data_ptr(), stream_ptr)
        assert rc == 0, rc
    dw.n_reads = n
    return go


def kernel_times(go, runs):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(runs):
            go()
        torch.cuda.synchronize()
    tot = {k: 0.0 for k in KERNELS}
    for ev in prof.events():
        for k in KERNELS:
            if k in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA:
                tot[k] += ev.device_time / 1000.0
    return {k: tot[k] / runs for k in KERNELS}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--lib", action="append", default=[], help="another build of libbrc_synth.so to time and compare")
    ap.add_argument("--bench", action="store_true", help="also run bench.py (C4) with resident windows and with --no-resident")
    args = ap.parse_args()

    import torch
    from bam_readcount_b200 import synth_cb as sc
    assert torch.cuda.is_available(), "synth_bench needs a CUDA device"
    name, pl = card()
    libs = [("tree", sc.load())] + [(p, C.CDLL(os.path.abspath(p))) for p in args.lib]
    for _, lib in libs[1:]:
        lib.brc_synth_fill_device.argtypes = sc.load().brc_synth_fill_device.argtypes
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream()
    out = {"card": name, "power_limit_w": pl, "runs": args.runs, "shapes": {}}
    for shape, (spec, contig, lo, hi) in shapes().items():
        n = spec.window_reads(lo, hi)
        dw = sc.DeviceWindow(spec, n + 256, dev)
        nbytes = n * sc.DeviceWindow.bytes_per_read()
        fills = [(label, fill_fn(lib, dw, contig, lo, hi, stream.cuda_stream)) for label, lib in libs]
        res = {label: [] for label, _ in fills}
        ref = None
        for label, go in fills:                       # warm-up, and every build writes the same bytes
            for _ in range(args.warmup):
                go()
            torch.cuda.synchronize()
            img = {k: v[: (n + 1) * 150].cpu() for k, v in dw.t.items() if k != "scratch"}
            if ref is None:
                ref = img
            else:
                res.setdefault("identical_to_tree", {})[label] = all(torch.equal(ref[k], img[k]) for k in ref)
        for _ in range(args.runs):                    # builds alternate, one fill each
            for label, go in fills:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                go()
                e1.record(stream)
                e1.synchronize()
                res[label].append(e0.elapsed_time(e1))
        entry = {"reads": n, "bytes": nbytes}
        for label, go in fills:
            ms = statistics.median(res[label])
            entry[label] = {"fill_ms_median": ms, "fill_ms_min": min(res[label]), "fill_ms_max": max(res[label]),
                            "write_gbs": nbytes / (ms / 1000.0) / 1e9, "kernel_ms": kernel_times(go, args.runs)}
        if "identical_to_tree" in res:
            entry["identical_to_tree"] = res["identical_to_tree"]
        out["shapes"][shape] = entry
        del dw
        torch.cuda.empty_cache()
    if args.bench:
        out["bench"] = {}
        for label, extra in (("c4_resident", []), ("c4_no_resident", ["--no-resident"])):
            p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--no-cpu-baseline", "--no-e2e-text"] + extra,
                               stdout=subprocess.PIPE, text=True)
            lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
            r = json.loads(lines[-1]) if lines else {"returncode": p.returncode}
            cfg, roof = r.get("config", {}), r.get("roofline", {})
            out["bench"][label] = {"ms_per_step": r.get("ms_per_step"), "value": r.get("value"), "gen_ms_per_window": cfg.get("gen_ms_per_window"),
                                   "windows_resident_rank0": cfg.get("windows_resident_rank0"), "k0_ms": roof.get("k0_ms"),
                                   "k1_ms": roof.get("k1_ms"), "parity": r.get("parity")}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
