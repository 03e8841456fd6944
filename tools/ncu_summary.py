"""Turn one `ncu --set full` capture (.ncu-rep, one kernel launch) into a markdown summary.

usage: python tools/ncu_summary.py prof_x.ncu-rep "title" > summary.md
"""
import csv
import io
import subprocess
import sys

KEYS = [
    ("gpu__time_duration.sum", "duration"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM throughput % of peak"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe active % (of active cycles)"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed", "tensor pipe active % (elapsed)"),
    ("sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "XU (MUFU) pipe %"),
    ("sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "FMA pipe %"),
    ("sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "ALU pipe %"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots active %"),
    ("l1tex__data_pipe_tc_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed", "tensor-core shared-memory wavefronts % of peak"),
    ("l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed", "LSU shared-memory wavefronts % of peak"),
    ("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "LSU shared-memory bank conflicts"),
    ("dram__bytes_read.sum", "DRAM bytes read"),
    ("dram__bytes_write.sum", "DRAM bytes written"),
    ("dram__bytes_read.sum.pct_of_peak_sustained_elapsed", "DRAM read % of peak"),
    ("lts__t_sector_hit_rate.pct", "L2 hit rate %"),
    ("launch__registers_per_thread", "registers / thread"),
    ("launch__shared_mem_per_block_dynamic", "dynamic shared memory / CTA"),
    ("launch__grid_size", "grid"),
    ("launch__block_size", "block"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy %"),
    ("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "stall: long scoreboard"),
    ("smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "stall: wait (fixed latency)"),
    ("smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "stall: short scoreboard"),
    ("smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio", "stall: MIO throttle"),
    ("smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "stall: barrier"),
    ("smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio", "stall: branch resolving"),
    ("smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio", "stall: math pipe throttle"),
]


def main():
    rep, title = sys.argv[1], sys.argv[2]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units, vals = rows[0], rows[1], rows[2]
    d = {h: (v, u) for h, u, v in zip(hdr, units, vals)}
    print(f"# {title}\n")
    print(f"kernel: `{d.get('Kernel Name', ('?', ''))[0]}`  — one launch, `ncu --set full --clock-control none`, source: `{rep.split('/')[-1]}`\n")
    print("| metric | value |\n|---|---|")
    for k, label in KEYS:
        if k in d and d[k][0] not in ("", "n/a"):
            print(f"| {label} (`{k}`) | {d[k][0]} {d[k][1]} |")


if __name__ == "__main__":
    main()
