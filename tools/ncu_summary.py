#!/usr/bin/env python3
"""Summarise an .ncu-rep (read here, no GPU needed) and a launch-list CSV into markdown.
usage: tools/ncu_summary.py <report.ncu-rep> [launches.csv]"""
import csv, io, subprocess, sys, collections

WANT = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
        "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_registers",
        "smsp__inst_executed.sum", "sm__inst_executed.avg.per_cycle_elapsed", "smsp__thread_inst_executed_per_inst_executed.ratio",
        "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
        "smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio", "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio", "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio", "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio"]


def main():
    rep = sys.argv[1]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    print(f"## ncu --set full: `{rep.split('/')[-1]}`\n")
    for r in rows[2:]:
        d = dict(zip(hdr, r))
        print(f"### {d.get('Kernel Name', '?')[:110]}\n")
        print("| metric | value | unit |\n|---|---:|---|")
        for w in WANT:
            if w in d:
                print(f"| {w} | {d[w]} | {units[hdr.index(w)]} |")
        try:
            t = float(d["gpu__time_duration.sum"]); u = units[hdr.index("gpu__time_duration.sum")]
            t_s = t * {"ns": 1e-9, "us": 1e-6, "usecond": 1e-6, "ms": 1e-3, "msecond": 1e-3, "s": 1, "second": 1}.get(u, 1e-9)
            rd = float(d["dram__bytes_read.sum"]) * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}[units[hdr.index("dram__bytes_read.sum")]]
            wr = float(d["dram__bytes_write.sum"]) * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}[units[hdr.index("dram__bytes_write.sum")]]
            print(f"\nDRAM traffic {(rd + wr) / 1e6:.1f} MB in {t_s * 1e3:.3f} ms = {(rd + wr) / t_s / 1e9:.0f} GB/s\n")
        except Exception as e:
            print(f"\n(traffic summary unavailable: {e})\n")
    if len(sys.argv) > 2:
        agg = collections.defaultdict(lambda: [0, 0.0])
        for r in csv.DictReader(l for l in open(sys.argv[2]) if l.startswith('"')):
            try:
                v = float(r["Metric Value"].replace(",", ""))
            except Exception:
                continue
            scale = {"ns": 1e-6, "us": 1e-3, "usecond": 1e-3, "ms": 1, "msecond": 1}.get(r["Metric Unit"], 1e-6)
            k = r["Kernel Name"].split("(")[0][:70]
            agg[k][0] += 1; agg[k][1] += v * scale
        tot = sum(v[1] for v in agg.values())
        print(f"## launch list `{sys.argv[2].split('/')[-1]}` (gpu__time_duration.sum; cold-cache, serialised: compare shares)\n")
        print("| kernel | launches | total ms | share |\n|---|---:|---:|---:|")
        for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            print(f"| {k} | {v[0]} | {v[1]:.3f} | {100 * v[1] / tot:.1f}% |")


if __name__ == "__main__":
    main()
