"""Summarise an .ncu-rep (from `ncu --set full`) into a small markdown table.
usage: ncu_summary.py REPORT.ncu-rep OUT.md "title" """
import csv, subprocess, sys

KEYS = [
    ("gpu__time_duration.sum", "duration"),
    ("launch__grid_size", "grid"), ("launch__block_size", "block"),
    ("launch__registers_per_thread", "registers/thread"),
    ("launch__shared_mem_per_block_dynamic", "dynamic smem/block"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy (% of max warps)"),
    ("dram__bytes_read.sum", "DRAM read"), ("dram__bytes_write.sum", "DRAM written"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "DRAM throughput (% peak)"),
    ("lts__t_sector_hit_rate.pct", "L2 hit rate"), ("l1tex__t_sector_hit_rate.pct", "L1 hit rate"),
    ("smsp__inst_executed.sum", "warp instructions"),
    ("smsp__thread_inst_executed_per_inst_executed.ratio", "active threads / warp instruction"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots busy"),
    ("sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "fma pipe instr (% peak)"),
    ("sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_elapsed", "fmaheavy (IMAD) pipe busy"),
    ("sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "alu pipe instr (% peak)"),
    ("sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "lsu pipe instr (% peak)"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe busy"),
    ("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smem bank conflicts"),
    ("l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "smem wavefronts"),
]
STALLS = "smsp__average_warps_issue_stalled_%s_per_issue_active.ratio"
STALL_NAMES = ["wait", "no_instruction", "math_pipe_throttle", "long_scoreboard", "short_scoreboard", "barrier",
               "dispatch_stall", "not_selected", "mio_throttle", "lg_throttle", "branch_resolving"]


def main():
    rep, out, title = sys.argv[1], sys.argv[2], sys.argv[3]
    txt = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(txt.splitlines()))
    hdr, units = rows[0], rows[1]
    with open(out, "w") as f:
        f.write(f"# {title}\n\nSource: `{rep.split('/')[-1]}` (`ncu --set full --clock-control none --import-source on`), "
                "read with `ncu -i ... --page raw --csv`.\n")
        for r in rows[2:]:
            name = r[hdr.index("Kernel Name")]
            f.write(f"\n## launch {r[hdr.index('ID')]}: `{name[:90]}`\n\n| metric | value |\n|---|---|\n")
            for k, label in KEYS:
                if k in hdr:
                    i = hdr.index(k)
                    f.write(f"| {label} (`{k}`) | {r[i]} {units[i]} |\n")
            f.write("\nWarp stall reasons (warps stalled per issue-active cycle):\n\n| reason | value |\n|---|---|\n")
            st = []
            for s in STALL_NAMES:
                k = STALLS % s
                if k in hdr:
                    st.append((float(r[hdr.index(k)].replace(",", "")), s))
            for v, s in sorted(st, reverse=True):
                f.write(f"| {s} | {v:.3f} |\n")
    print(open(out).read())


if __name__ == "__main__":
    main()
