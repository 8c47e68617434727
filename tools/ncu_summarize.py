"""Turn ncu output into text summaries.

  python tools/ncu_summarize.py launches <launches.csv>          # per-kernel totals/shares of a `--metrics gpu__time_duration.sum` list
  python tools/ncu_summarize.py full <report.ncu-rep>            # the metrics DESIGN.md quotes from one `--set full` capture
"""
import csv, io, subprocess, sys
from collections import defaultdict


def launches(path):
    rows = [r for r in csv.reader(l for l in open(path) if l.startswith('"'))]
    hdr = rows[0]; ix = {h: i for i, h in enumerate(hdr)}
    tot = defaultdict(float); cnt = defaultdict(int)
    for r in rows[1:]:
        if r[ix["Metric Name"]] != "gpu__time_duration.sum":
            continue
        v = float(r[ix["Metric Value"]].replace(",", ""))
        unit = r[ix["Metric Unit"]]
        ms = v * {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3}.get(unit, 1e-6)
        k = r[ix["Kernel Name"]]
        tot[k] += ms; cnt[k] += 1
    allms = sum(tot.values())
    print(f"{'kernel':72s} {'launches':>8s} {'total ms':>10s} {'share':>7s}")
    for k, v in sorted(tot.items(), key=lambda kv: -kv[1])[:16]:
        print(f"{k[:72]:72s} {cnt[k]:8d} {v:10.3f} {100 * v / allms:6.1f}%")
    print(f"{'(all kernels)':72s} {sum(cnt.values()):8d} {allms:10.3f}")


WANT = ["gpu__time_duration.sum", "sm__cycles_elapsed.avg", "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
        "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_shared_mem", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_tensor.sum",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio"]


def full(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units, vals = rows[0], rows[1], rows[2]
    ix = {h: i for i, h in enumerate(hdr)}
    print("kernel:", vals[ix["Kernel Name"]])
    for m in WANT:
        if m in ix:
            print(f"  {m:88s} {vals[ix[m]]:>18s} {units[ix[m]]}")


if __name__ == "__main__":
    {"launches": launches, "full": full}[sys.argv[1]](sys.argv[2])
