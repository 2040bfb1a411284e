#!/usr/bin/env python
"""Turn gpurun_out/{prof_k0,prof_k1}_<tag>.ncu-rep + launches_<tag>.csv into committed text under profiles/."""
import csv, io, json, os, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
        "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "smsp__thread_inst_executed_per_inst_executed.ratio",
        "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio", "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum"]


def raw(rep):
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    return {h: (u, v) for h, u, v in zip(rows[0], rows[1], rows[2])}, rows[2][rows[0].index("Kernel Name")] if "Kernel Name" in rows[0] else ""


def to_bytes(v, u):
    f = float(v)
    return f * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(u, 1)


def main(tag, session=None):
    """tag: name of the summary (profiles/ncu_<tag>.md).  session: directory under gpurun_out/ written by tools/gpu_session.sh
    (prof_*.ncu-rep, launches_c4.csv); default = the round-1 layout (gpurun_out/prof_k?_<tag>.ncu-rep)."""
    import glob
    out = [f"# ncu summary {tag}", "", "Command: `tools/gpu_session.sh` — `ncu --set full --clock-control none --import-source on -k regex:<kernel> -s 4 -c 1 python bench.py "
           "--config c3 --steps 2 --warmup 3 ...` (K0/K1 on the resident 10 Mb window; deep: `--config c5`; inflate: the span parity test), 1 H100.", ""]
    traffic = {}
    if session:
        reps = sorted(glob.glob(os.path.join(ROOT, "gpurun_out", session, "prof_*.ncu-rep")))
    else:
        reps = [os.path.join(ROOT, "gpurun_out", f"prof_{k}_{tag}.ncu-rep") for k in ("k0", "k1")]
    for rep in reps:
        if not os.path.exists(rep):
            continue
        m, kname = raw(rep)
        name = kname.split("(")[0].replace("void ", "").replace("brc::", "").replace("<", "_").replace(">", "").strip() or os.path.basename(rep)
        if "pileup_kernel" in name:
            name = "pileup_kernel"
        out += [f"## {name}  ({os.path.basename(rep)})", "", "| metric | unit | value |", "|---|---|---|"]
        for key in KEYS + ["smsp__sass_inst_executed_op_local_ld.sum", "launch__shared_mem_per_block_dynamic"]:
            if key in m:
                out.append(f"| {key} | {m[key][0]} | {m[key][1]} |")
        rd = to_bytes(m["dram__bytes_read.sum"][1], m["dram__bytes_read.sum"][0])
        wr = to_bytes(m["dram__bytes_write.sum"][1], m["dram__bytes_write.sum"][0])
        traffic[name] = {"dram_bytes_read": rd, "dram_bytes_write": wr, "traffic": rd + wr, "duration": m["gpu__time_duration.sum"][1] + " " + m["gpu__time_duration.sum"][0]}
        out += ["", f"DRAM traffic per launch: read {rd/1e6:.1f} MB + write {wr/1e6:.1f} MB = **{(rd+wr)/1e6:.1f} MB**", ""]
    lc = os.path.join(ROOT, "gpurun_out", session, "launches_c4.csv") if session else os.path.join(ROOT, "gpurun_out", f"launches_{tag}.csv")
    if os.path.exists(lc):
        rows = [r for r in csv.reader(open(lc)) if len(r) > 5 and r[0].isdigit()]
        agg = {}
        for r in rows:
            kn = r[4].split("(")[0]
            agg.setdefault(kn, []).append(float(r[-1]))
        tot = sum(sum(v) for v in agg.values())
        out += ["## launch list of `bench.py` (C4, one contig) under `ncu --metrics gpu__time_duration.sum` (ns; cold-cache, serialised — compare shares)", "",
                "| kernel | launches | mean ns | share |", "|---|---|---|---|"]
        for kn, v in sorted(agg.items(), key=lambda kv: -sum(kv[1])):
            out.append(f"| {kn} | {len(v)} | {sum(v)/len(v):.0f} | {100*sum(v)/tot:.1f}% |")
        import shutil
        shutil.copy(lc, os.path.join(ROOT, "profiles", f"launches_{tag}.csv"))
    os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
    open(os.path.join(ROOT, "profiles", f"ncu_{tag}.md"), "w").write("\n".join(out) + "\n")
    json.dump({"tag": tag, **traffic}, open(os.path.join(ROOT, "profiles", f"traffic_{tag}.json"), "w"), indent=1)
    print("\n".join(out[:14]))


if __name__ == "__main__":
    main(*sys.argv[1:3])
