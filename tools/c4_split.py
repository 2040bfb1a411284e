"""Where one C4 genome pass spends its device time, kernel by kernel; prints one JSON line.

Two measurements, in one process:
  isolated  on one C4 window (a middle window of contig 0) and one contig change, each step on one stream behind a device
            synchronise, --reps times under torch.profiler: the median time of every kernel it launches — the generator's
            count, scan and fill kernels, the reference generation (synth_ref_kernel), the reference encode (the memset and
            ref_encode_kernel of brc_set_reference_device) and the engine's init_tiles, K0 (read_precompute_kernel) and K1
            (pileup_kernel).
  one pass  bench.py's C4 loop over every window on three WindowRunners (windows dealt round-robin, every window regenerated,
            as with bench.py --no-resident): the launches of each kernel that one pass makes, counted by torch.profiler,
            and the pass time (CUDA events, profiler off).
Median x launches per pass is each kernel's share of a pass.  The card's name and power limit are printed with the numbers.

    python tools/c4_split.py [--reps 30] [--contigs 24]
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

KERNELS = ("synth_count_kernel", "synth_scan_kernel", "synth_fill_kernel", "synth_ref_kernel", "ref_encode_kernel",
           "init_tiles_kernel", "read_precompute_kernel", "pileup_kernel")


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], text=True).strip()
    except Exception:
        pl = None
    return name, pl


def kernel_key(name: str) -> str:
    for k in KERNELS:
        if k in name:
            return k
    return "memset" if "memset" in name.lower() else name.split("(")[0][-60:]


def profiled(go):
    """{kernel: [device ms of each launch]} of what go() enqueues."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        go()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            out.setdefault(kernel_key(ev.name), []).append(ev.device_time / 1000.0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--contigs", type=int, default=24)
    args = ap.parse_args()
    import torch
    from bam_readcount_b200 import stream as st
    from bam_readcount_b200 import synth_cb
    from bench import CONFIGS

    cfg = CONFIGS["c4"]
    spec = synth_cb.Spec(seed=1234, mode=synth_cb.WGS, n_libs=8, contig_len=cfg["contig_blocks"] * synth_cb.BLOCK_BP, n_contigs=args.contigs)
    windows = st.wgs_windows(spec, cfg["windows_per_contig"])
    device = torch.device("cuda", 0)
    max_reads = max(spec.window_reads(w.blk_lo, w.blk_hi) for w in windows)
    runners = [st.WindowRunner(spec, max_reads, device, cfg["flags"]) for _ in range(3)]

    def one_pass():
        for k, w in enumerate(windows):
            runners[k % 3].launch(w)
        cur = torch.cuda.current_stream()
        for r in runners:
            cur.wait_stream(r.stream)

    # ---- one pass: launches per kernel, and the pass time ----
    one_pass()                      # warm-up: modules loaded, buffers allocated, runners on the last contig as in a steady pass
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    one_pass()
    ev1.record()
    torch.cuda.synchronize()
    pass_ms = ev0.elapsed_time(ev1)
    per_pass = {k: len(v) for k, v in profiled(one_pass).items()}
    for r in runners:
        r.busy = False

    # ---- isolated: one window and one contig change on runner 0's stream, each step behind a synchronise ----
    r0 = runners[0]
    w0 = windows[len([w for w in windows if w.contig == 0]) // 2]
    r0.launch(w0)
    torch.cuda.synchronize()
    L = spec.contig_len
    ascii_buf = torch.empty(L + 64, dtype=torch.uint8, device=device)
    sp = r0.stream.cuda_stream
    steps = {
        "generator": lambda: r0.dw.fill(w0.contig, w0.blk_lo, w0.blk_hi, sp),
        "reference": lambda: synth_cb.load().brc_synth_ref_device(C.byref(spec.c), 1, 0, L, ascii_buf.data_ptr(), sp),
        "encode": lambda: r0.eng.set_reference_device(1, "chr2", L, 0, ascii_buf.data_ptr(), L, sp),
        "engine": lambda: r0.eng.run_device(r0.dw.c_batch(), None, sp),
    }

    def isolated():
        for _ in range(args.reps):
            for go in steps.values():
                go()
                torch.cuda.synchronize()
    for go in steps.values():
        go()
    times = profiled(isolated)
    kernels = {}
    for k in sorted(set(times) | set(per_pass)):
        med = statistics.median(times[k]) if k in times else None
        n = per_pass.get(k, 0)
        kernels[k] = {"median_ms": round(med, 4) if med is not None else None, "launches_per_pass": n,
                      "ms_per_pass": round(med * n, 1) if med is not None else None}
    for r in runners:
        r.close()
    name, pl = card()
    line = {"tool": "c4_split", "gpu": name, "power_limit_w": pl, "contigs": args.contigs, "windows_per_pass": len(windows),
            "window_reads": spec.window_reads(w0.blk_lo, w0.blk_hi), "reps": args.reps, "pass_ms_all_windows_regenerated": round(pass_ms, 1),
            "kernels": kernels}
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    sys.exit(main())
