"""Turns an .ncu-rep into a small text summary:
key raw metrics + the top source lines by instructions and by stall samples.

    python scripts/ncu_summary.py prof_inflate.ncu-rep out/inflate
"""
import csv
import io
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "launch__grid_size", "launch__block_size",
        "launch__registers_per_thread", "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_registers",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum", "smsp__thread_inst_executed.sum",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__average_warp_latency_per_inst_issued.ratio",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
        "dram__throughput.avg.pct_of_peak_sustained_elapsed", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__t_sector_hit_rate.pct", "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum",
        "l1tex__t_sectors_pipe_lsu_mem_global_op_ld_lookup_hit.sum", "l1tex__t_sectors_pipe_lsu_mem_global_op_st.sum",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
        "sm__cycles_elapsed.max", "smsp__cycles_active.avg"]


def ncu(args):
    return subprocess.run(["ncu"] + args, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True).stdout


def main():
    rep, out = sys.argv[1], sys.argv[2]
    raw = list(csv.reader(io.StringIO(ncu(["-i", rep, "--page", "raw", "--csv"]))))
    hdr, units = raw[0], raw[1]
    lines = ["# ncu summary of %s" % rep, ""]
    for row in raw[2:]:
        d = dict(zip(hdr, row))
        lines.append("## kernel: %s  (launch id %s)" % (d.get("Kernel Name", "?"), d.get("ID", "?")))
        lines.append("")
        lines.append("| metric | value | unit |")
        lines.append("|---|---|---|")
        for k in KEYS:
            if k in d:
                lines.append("| %s | %s | %s |" % (k, d[k], units[hdr.index(k)]))
        lines.append("")
    src = list(csv.reader(io.StringIO(ncu(["-i", rep, "--page", "source", "--csv", "--print-source", "cuda,sass"]))))
    h = None
    for i, r in enumerate(src):
        if r and r[0] == "Line No":
            h = i
            break
    if h is not None:
        hdr2 = src[h]
        ie, isamp, ithr = hdr2.index("Instructions Executed"), hdr2.index("# Samples"), hdr2.index("Thread Instructions Executed")
        data = []
        for r in src[h + 1:]:
            if len(r) <= ie or not r[0]:
                continue
            try:
                data.append((int(r[ie]), int(r[isamp]), int(r[ithr]), r[0], r[1].strip()[:100]))
            except ValueError:
                pass
        tot = sum(d[0] for d in data) or 1
        tots = sum(d[1] for d in data) or 1
        for title, key in (("Top source lines by warp instructions executed", 0), ("Top source lines by stall samples", 1)):
            lines += ["## " + title, "", "| % inst | % samples | active threads/inst | line | source |", "|---|---|---|---|---|"]
            for n, s, t, ln, code in sorted(data, key=lambda d: d[key], reverse=True)[:25]:
                lines.append("| %.1f | %.1f | %.1f | %s | `%s` |" % (100.0 * n / tot, 100.0 * s / tots, t / max(1, n), ln, code.replace("|", "\\|")))
            lines.append("")
    open(out + ".md", "w").write("\n".join(lines) + "\n")
    print("wrote", out + ".md")


if __name__ == "__main__":
    main()
