#!/usr/bin/env python
"""Summarises an ncu launch list (CSV) or an ncu report into a small markdown file.

    python tools/summarize_ncu.py launches <launches.csv> <out.md>
    python tools/summarize_ncu.py report   <report.ncu-rep> <out.md>
"""
import collections
import csv
import io
import subprocess
import sys

METRICS = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
    "launch__shared_mem_per_block_dynamic", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "sm__maximum_warps_per_active_cycle_pct", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed.sum.per_cycle_active", "smsp__inst_executed.sum",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
    "smsp__thread_inst_executed_per_inst_executed.ratio", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct",
    "smsp__warps_eligible.avg.per_cycle_active", "smsp__warp_issue_stalled_math_pipe_throttle_per_warp_active.pct",
    "smsp__warp_issue_stalled_long_scoreboard_per_warp_active.pct",
    "smsp__warp_issue_stalled_short_scoreboard_per_warp_active.pct",
    "smsp__warp_issue_stalled_wait_per_warp_active.pct", "smsp__warp_issue_stalled_not_selected_per_warp_active.pct",
    "smsp__warp_issue_stalled_branch_resolving_per_warp_active.pct",
]


def launches(src, dst):
    rows = list(csv.reader(open(src)))
    hi = [i for i, r in enumerate(rows) if r and r[0] == "ID"][0]
    hdr, data = rows[hi], rows[hi + 1:]
    ki, vi, ui = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    tot, cnt = collections.Counter(), collections.Counter()
    for r in data:
        if len(r) <= vi:
            continue
        v = float(r[vi].replace(",", ""))
        v *= {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3}.get(r[ui], 1.0)
        name = r[ki].split("(")[0].replace("void ", "")
        tot[name] += v
        cnt[name] += 1
    T = sum(tot.values())
    with open(dst, "w") as f:
        f.write(f"# ncu launch list ({src}): gpu__time_duration.sum per kernel\n\n")
        f.write("Cold-cache, serialised replays: compare SHARES, not absolutes. Includes the torch kernels that\n"
                "generate the synthetic inputs (native::*, at_cuda_detail::*), which are outside the timed region.\n\n")
        f.write(f"total {T:.3f} ms over {sum(cnt.values())} launches\n\n| ms | share | launches | kernel |\n|---:|---:|---:|---|\n")
        for k, v in tot.most_common(40):
            f.write(f"| {v:.3f} | {100 * v / T:.1f}% | {cnt[k]} | `{k[:110]}` |\n")
        ours = {k: v for k, v in tot.items() if k.startswith("b200::") or "CUB_" in k}
        To = sum(ours.values())
        f.write(f"\n## engine kernels only (b200::* and its CUB calls): {To:.3f} ms\n\n| ms | share | launches | kernel |\n|---:|---:|---:|---|\n")
        for k, v in sorted(ours.items(), key=lambda kv: -kv[1]):
            f.write(f"| {v:.3f} | {100 * v / To:.1f}% | {cnt[k]} | `{k[:110]}` |\n")


def trie(src, dst):
    """`ncu -i rep --page raw --csv` of the node kernels of one C3 build -> one row per launch."""
    rows = list(csv.reader(open(src)))
    hdr, data = rows[0], rows[2:]
    col = {h: i for i, h in enumerate(hdr)}
    cols = [("Kernel Name", "kernel"), ("launch__grid_size", "grid"), ("gpu__time_duration.sum", "ms"),
            ("launch__registers_per_thread", "regs"), ("launch__shared_mem_per_block_dynamic", "dyn smem KB"),
            ("smsp__inst_executed.sum", "warp inst"), ("smsp__thread_inst_executed_per_inst_executed.ratio", "active thr/warp"),
            ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps active %"),
            ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue %"),
            ("sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "ALU pipe %"),
            ("dram__bytes_read.sum", "DRAM rd"), ("dram__bytes_write.sum", "DRAM wr"),
            ("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "stall: long scoreboard"),
            ("smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio", "stall: math pipe")]
    units = rows[1]
    out = ["# ncu --set full, node kernels of one C3 build (1M accounts x 16 slots), round 2", "",
           "One row per launch in launch order (storage forest, then the account trie).  Durations are ncu replays (cold caches,",
           "serialised).  `leaf_storage_kernel` is the register-path storage leaf kernel (no shared-memory strip).", "",
           "| " + " | ".join(n for _, n in cols) + " |", "|" + "---|" * len(cols)]
    total = 0.0
    for r in data:
        vals = []
        for h, _ in cols:
            v = r[col[h]] if h in col else ""
            if h == "Kernel Name":
                v = "`" + v.split("(")[0].replace("void ", "") + "`"
            elif h == "launch__shared_mem_per_block_dynamic":
                v = f"{float(v) / 1024:.1f}" if units[col[h]] == "byte/block" else v
            elif h in ("dram__bytes_read.sum", "dram__bytes_write.sum"):
                u = units[col[h]]
                f = float(v) * {"Gbyte": 1000, "Mbyte": 1, "Kbyte": 1e-3, "byte": 1e-6}.get(u, 1)
                v = f"{f:.1f} MB"
            else:
                try:
                    fv = float(v)
                    v = f"{fv:.3f}" if h == "gpu__time_duration.sum" else (f"{fv:.0f}" if fv > 1000 else f"{fv:.1f}")
                except ValueError:
                    pass
            vals.append(v)
        total += float(r[col["gpu__time_duration.sum"]])
        out.append("| " + " | ".join(vals) + " |")
    out += ["", f"sum of the node kernels above: {total:.3f} ms"]
    open(dst, "w").write("\n".join(out) + "\n")


def report(src, dst):
    out = subprocess.run(["ncu", "-i", src, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    ki = hdr.index("Kernel Name")
    with open(dst, "w") as f:
        f.write(f"# ncu --set full summary of {src}\n\n")
        for r in data:
            gi = hdr.index("Grid Size") if "Grid Size" in hdr else None
            f.write(f"## `{r[ki][:90]}` grid {r[gi] if gi is not None else ''}\n\n| metric | value | unit |\n|---|---:|---|\n")
            for m in METRICS:
                if m in hdr:
                    i = hdr.index(m)
                    f.write(f"| {m} | {r[i]} | {units[i]} |\n")
            f.write("\n")


if __name__ == "__main__":
    {"launches": launches, "report": report, "trie": trie}[sys.argv[1]](sys.argv[2], sys.argv[3])
