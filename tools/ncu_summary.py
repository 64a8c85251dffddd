#!/usr/bin/env python
"""Summarises an .ncu-rep (read here with `ncu -i ... --page raw --csv`) into markdown tables, and prints
the DRAM traffic of the compositing kernels (bench.py reads it from profiles/roofline_traffic.json when present).

    python tools/ncu_summary.py out/prof.ncu-rep out/ncu.md "title"
"""
import csv
import io
import json
import subprocess
import sys

KEEP = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "launch__registers_per_thread",
    "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_registers",
    "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_warps", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "smsp__inst_executed.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "smsp__thread_inst_executed_per_inst_executed.ratio",
    "lts__t_sectors_op_red.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
]


def main():
    rep, out, title = sys.argv[1], sys.argv[2], sys.argv[3]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    name_i = hdr.index("Kernel Name")
    lines = [f"# {title}", ""]
    traffic = {}
    for r in data:
        lines += [f"## {r[name_i][:90]}", "", "| metric | value | unit |", "|---|---|---|"]
        vals = {}
        for k in KEEP:
            if k in hdr:
                i = hdr.index(k)
                vals[k] = (r[i], units[i])
                lines.append(f"| {k} | {r[i]} | {units[i]} |")
        # the eight largest warp-stall reasons (warps stalled per issue-active cycle)
        stalls = []
        for i, h in enumerate(hdr):
            if "issue_stalled" in h and h.endswith("_per_issue_active.ratio"):
                try:
                    stalls.append((float(r[i].replace(",", "")), h.replace("smsp__average_warps_issue_stalled_", "").replace("_per_issue_active.ratio", "")))
                except ValueError:
                    pass
        for v, h in sorted(stalls, reverse=True)[:8]:
            lines.append(f"| stall: {h} | {v:.3f} | warps / issue-active cycle |")
        for k in ("l1tex__data_bank_conflicts_pipe_lsu_mem_shared_op_ld.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared_op_st.sum",
                  "lts__t_sectors_op_atom.sum", "lts__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__throughput.avg.pct_of_peak_sustained_active",
                  "smsp__inst_executed_op_shared_ld.sum", "smsp__inst_executed_op_shared_st.sum", "smsp__inst_executed_op_global_red.sum",
                  "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
                  "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active"):
            if k in hdr:
                i = hdr.index(k)
                lines.append(f"| {k} | {r[i]} | {units[i]} |")
        lines.append("")
        try:
            def to_bytes(k):
                v, u = vals[k]
                v = float(v.replace(",", ""))
                return v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}[u]
            traffic[r[name_i].split("(")[0]] = to_bytes("dram__bytes_read.sum") + to_bytes("dram__bytes_write.sum")
        except Exception:
            pass
    open(out, "w").write("\n".join(lines))
    print(json.dumps(traffic, indent=1))


if __name__ == "__main__":
    main()
