"""Condense one kernel of an ncu capture into a JSON summary.
    python tools/ncu_summary.py <report.ncu-rep> <kernel-name substring> <out.json> ["free-text note"]
Reads `ncu -i <rep> --page raw --csv`; the first launch whose name contains the substring is summarised."""
import csv, io, json, subprocess, sys

KEEP = [
    "gpu__time_duration.sum", "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__warps_active.avg.per_cycle_active", "launch__registers_per_thread",
    "launch__grid_size", "launch__block_size", "launch__waves_per_multiprocessor", "launch__shared_mem_per_block_dynamic",
    "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_registers", "launch__occupancy_limit_warps",
    "dram__bytes_read.sum", "dram__bytes_write.sum", "lts__t_bytes.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
    "smsp__thread_inst_executed_per_inst_executed.ratio", "smsp__average_warp_latency_per_inst_issued.ratio",
    "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
    "smsp__sass_thread_inst_executed_op_ffma_pred_on.sum.per_cycle_elapsed", "smsp__sass_thread_inst_executed_op_fadd_pred_on.sum.per_cycle_elapsed",
    "smsp__sass_thread_inst_executed_op_fmul_pred_on.sum.per_cycle_elapsed", "smsp__cycles_elapsed.avg",
    "l1tex__t_requests_pipe_lsu_mem_local_op_ld.sum", "l1tex__t_requests_pipe_lsu_mem_local_op_st.sum",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared_op_ld.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared_op_st.sum", "sm__cycles_elapsed.max",
]
STALLS = "smsp__average_warps_issue_stalled_%s_per_issue_active.ratio"
for s in ("wait", "short_scoreboard", "long_scoreboard", "no_instruction", "not_selected", "branch_resolving", "dispatch_stall", "math_pipe_throttle",
          "barrier", "mio_throttle", "lg_throttle", "imc_miss", "membar", "sleeping", "drain"):
    KEEP.append(STALLS % s)


def main():
    rep, pat, out = sys.argv[1:4]
    note = sys.argv[4] if len(sys.argv) > 4 else ""
    txt = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(txt)))
    hdr, units = rows[0], rows[1]
    ik = hdr.index("Kernel Name")
    row = next(r for r in rows[2:] if pat in r[ik])
    d = {"kernel": row[ik], "capture": rep.split("/")[-1]}
    for k in KEEP:
        if k in hdr:
            i = hdr.index(k)
            d[k] = (row[i] + " " + units[i]).strip()
    f = lambda k: float(d[k].split()[0].replace(",", "")) if k in d else 0.0
    pc = "smsp__sass_thread_inst_executed_op_%s_pred_on.sum.per_cycle_elapsed"
    flop = (2 * f(pc % "ffma") + f(pc % "fadd") + f(pc % "fmul")) * f("smsp__cycles_elapsed.avg")
    if flop:
        d["fp32_flop_per_launch (2*FFMA+FADD+FMUL thread-instructions)"] = flop
    if note:
        d["note"] = note
    json.dump(d, open(out, "w"), indent=1)
    print(json.dumps(d, indent=1))


if __name__ == "__main__":
    main()
