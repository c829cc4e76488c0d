#!/usr/bin/env python
"""ncu_summary.py REPORT.ncu-rep "title" "command" > summary.md — the metrics the roofline discussion needs, from one
`ncu --set full` capture (read with `ncu -i ... --page raw --csv`; works on a machine without a GPU)."""
import csv
import subprocess
import sys

rep, title, cmd = sys.argv[1], sys.argv[2], (sys.argv[3] if len(sys.argv) > 3 else "")
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units = rows[0], rows[1]
print(f"# ncu --set full summary: {title}\n")
if cmd:
    print(f"Command (1 GPU): `{cmd}`\n")
print("Profiler timings are cold-cache / serialised; bench values are never taken under ncu.\n")
KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__bytes.sum.per_second",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "launch__occupancy_limit_registers",
        "launch__occupancy_limit_shared_mem", "smsp__inst_executed.sum", "smsp__inst_executed.min", "smsp__inst_executed.max",
        "smsp__inst_executed.avg", "smsp__cycles_active.avg", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smsp__warps_eligible.avg.per_cycle_active",
        "smsp__inst_executed_op_local_ld.sum", "smsp__inst_executed_op_local_st.sum"]
for r in rows[2:]:
    d = dict(zip(hdr, r))
    u = dict(zip(hdr, units))
    print(f"## {d.get('Kernel Name', '?')}  grid {d.get('Grid Size', '')} block {d.get('Block Size', '')}\n")
    print("| metric | value | unit |\n|---|---|---|")
    for k in KEYS:
        if k in d and d[k] != "":
            print(f"| {k} | {d[k]} | {u.get(k, '')} |")
    print("\nWarp stall reasons (warps stalled per issue-active cycle):\n\n| reason | ratio |\n|---|---|")
    st = [(k.split("issue_stalled_")[1].split("_per_issue")[0], float(d[k])) for k in hdr if "smsp__average_warps_issue_stalled" in k and k.endswith("_per_issue_active.ratio") and d[k] not in ("", "n/a")]
    for name, v in sorted(st, key=lambda x: -x[1]):
        if v >= 0.01:
            print(f"| {name} | {v:.3f} |")
    try:
        rd, wr = float(d["dram__bytes_read.sum"]), float(d["dram__bytes_write.sum"])
        print(f"\nDRAM traffic per launch: read {rd} {u['dram__bytes_read.sum']} + write {wr} {u['dram__bytes_write.sum']}.")
        alu = float(d["sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active"])
        print(f"ALU pipe {alu:.1f} % busy (the pipe issues one warp instruction per two cycles: this is LOP3 / mask / XOR work).")
    except Exception:
        pass
    print()
