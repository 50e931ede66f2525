"""Summarise Nsight Compute captures into small text files (no GPU needed).

    python tools/ncu_summary.py launches launches.csv > launches.txt
    python tools/ncu_summary.py full prof_gemm.ncu-rep > ncu_gemm.txt
"""
import collections
import csv
import re
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
    "launch__shared_mem_per_block_dynamic", "sm__cycles_elapsed.avg", "sm__cycles_elapsed.avg.per_second",
    "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed",
    "sm__pipe_tc_cycles_active.avg.pct_of_peak_sustained_elapsed",
    "sm__mem_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed",
    "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_elapsed",
    "sm__inst_executed_pipe_tmem.avg.pct_of_peak_sustained_active",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
    "lts__t_bytes.sum", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
]


def launches(path):
    lines = [l for l in open(path) if not l.startswith("==")]
    tot, cnt = collections.defaultdict(float), collections.Counter()
    for row in csv.DictReader(lines):
        if row.get("Metric Name") != "gpu__time_duration.sum":
            continue
        name = re.sub(r"\(.*", "", row["Kernel Name"])
        v = float(row["Metric Value"].replace(",", ""))
        v *= {"ns": 1.0, "us": 1e3, "ms": 1e6, "s": 1e9}.get(row["Metric Unit"], 1.0)
        tot[name] += v
        cnt[name] += 1
    T = sum(tot.values())
    print(f"# ncu --metrics gpu__time_duration.sum --clock-control none (cold-cache, serialised): {sum(cnt.values())} launches, "
          f"{T / 1e6:.3f} ms total")
    print(f"# {'ms':>10} {'share':>6} {'n':>6} {'avg us':>9}  kernel")
    for k, v in sorted(tot.items(), key=lambda kv: -kv[1]):
        print(f"{v / 1e6:12.3f} {100 * v / T:5.1f}% {cnt[k]:6d} {v / cnt[k] / 1e3:9.1f}  {k[:100]}")


def full(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    print(f"# ncu --set full --clock-control none : {path}")
    for row in rows[2:]:
        d = dict(zip(hdr, row))
        u = dict(zip(hdr, units))
        print(f"\n== {d.get('Kernel Name', '?')}")
        for k in KEYS:
            if k in d and d[k] not in ("", "n/a"):
                print(f"   {k:100s} {d[k]} {u.get(k, '')}")


if __name__ == "__main__":
    {"launches": launches, "full": full}[sys.argv[1]](sys.argv[2])
