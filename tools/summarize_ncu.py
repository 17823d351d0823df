#!/usr/bin/env python
"""Turn Nsight Compute outputs into small text summaries.

    python tools/summarize_ncu.py launches launches.csv          > launches.md
    python tools/summarize_ncu.py kernel   prof_recon.ncu-rep    > reconstruct.md
    python tools/summarize_ncu.py lines    prof_walk.ncu-rep 25  >> walk.md   # hottest source lines
"""
import csv
import io
import subprocess
import sys
from collections import defaultdict

KEYS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "smsp__inst_executed.sum", "smsp__thread_inst_executed_per_inst_executed.ratio",
    "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "launch__waves_per_multiprocessor",
    "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_warps",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
    "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum", "l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
]


def launches(path):
    rows = [r for r in csv.reader(open(path)) if r and not r[0].startswith("==")]
    hdr = rows[0]
    ik, im, iv = hdr.index("Kernel Name"), hdr.index("Metric Name"), hdr.index("Metric Value")
    iu = hdr.index("Metric Unit")
    tot = defaultdict(float)
    cnt = defaultdict(int)
    for r in rows[1:]:
        if r[im] != "gpu__time_duration.sum":
            continue
        v = float(r[iv].replace(",", ""))
        v *= {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6, "nsecond": 1e-3, "usecond": 1.0, "msecond": 1e3, "second": 1e6}.get(r[iu], 1.0)
        name = r[ik].split("(")[0].split("::")[-1]
        tot[name] += v
        cnt[name] += 1
    total = sum(tot.values())
    print("| kernel | launches | total us | avg us | share |")
    print("|---|---:|---:|---:|---:|")
    for k, v in sorted(tot.items(), key=lambda kv: -kv[1]):
        print(f"| {k} | {cnt[k]} | {v:.0f} | {v / cnt[k]:.1f} | {100 * v / total:.1f} % |")
    print(f"\n{sum(cnt.values())} launches, {total / 1e3:.1f} ms of kernel time (ncu: serialised, cold caches; compare shares, not absolutes)")


def kernel(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    ik = hdr.index("Kernel Name")
    print(f"source: {path}; {len(data)} launch(es) of {data[0][ik].split('(')[0]}\n")
    print("| metric | unit | " + " | ".join(f"launch {i}" for i in range(len(data))) + " |")
    print("|---|---|" + "---:|" * len(data))
    for k in KEYS:
        if k in hdr:
            i = hdr.index(k)
            print(f"| {k} | {units[i]} | " + " | ".join(r[i] for r in data) + " |")
    print("\nwarps stalled per issued instruction, by reason (smsp__average_warps_issue_stalled_*_per_issue_active, > 0.2):\n")
    for i, h in enumerate(hdr):
        if "issue_stalled" in h and h.endswith("per_issue_active.ratio") and "not_issued" not in h:
            v = [float(r[i] or 0) for r in data]
            if max(v) > 0.2:
                print("* " + h.split("stalled_")[1].replace("_per_issue_active.ratio", "") + ": " + ", ".join(f"{x:.2f}" for x in v))
    print("\nwarp issue stall reasons (% of active warps, > 3 %):\n")
    for i, h in enumerate(hdr):
        if "warp_issue_stalled" in h and h.endswith("per_warp_active.pct"):
            v = [float(r[i] or 0) for r in data]
            if max(v) > 3:
                print("* " + h.replace("smsp__warp_issue_stalled_", "").replace("_per_warp_active.pct", "") + ": " + ", ".join(f"{x:.1f}" for x in v))


def lines(path, top=25):
    """The source lines (needs -lineinfo + --import-source on) with the most warp-stall samples, summed over the launches."""
    out = subprocess.run(["ncu", "-i", path, "--page", "source", "--print-source", "cuda,sass", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    keys = ["# Samples", "Instructions Executed", "stall_long_sb", "stall_wait", "stall_short_sb", "stall_branch_resolving", "stall_math",
            "stall_barrier", "stall_not_selected"]
    cur, hdr, agg = None, None, {}
    for r in rows:
        if len(r) == 2 and r[0] == "File Path":
            cur = r[1].split("/")[-1]
        elif len(r) > 5 and r[0] == "Line No":
            hdr = r
        elif hdr and len(r) == len(hdr) and r[0] != "":
            d = dict(zip(hdr, r))
            try:
                v = [int(d[k]) for k in keys]
            except (KeyError, ValueError):
                continue
            k = (cur, r[0], r[1].strip()[:110])
            agg[k] = [a + b for a, b in zip(agg.get(k, [0] * len(keys)), v)]
    tot = sum(v[0] for v in agg.values()) or 1
    toti = sum(v[1] for v in agg.values()) or 1
    print(f"\nhottest source lines of {path} (share of warp-stall samples | of warp instructions | dominant stall reasons in samples):\n")
    print("| samples | instr | long sb | wait | short sb | branch | math | barrier | not sel | line |")
    print("|---:|---:|---:|---:|---:|---:|---:|---:|---:|---|")
    for k, v in sorted(agg.items(), key=lambda kv: -kv[1][0])[:int(top)]:
        print(f"| {100 * v[0] / tot:.1f} % | {100 * v[1] / toti:.1f} % | " + " | ".join(str(x) for x in v[2:]) + f" | `{k[0]}:{k[1]}` `{k[2]}` |")


if __name__ == "__main__":
    {"launches": launches, "kernel": kernel, "lines": lines}[sys.argv[1]](*sys.argv[2:])
