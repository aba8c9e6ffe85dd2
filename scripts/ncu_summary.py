#!/usr/bin/env python
"""Turn ncu CSV exports into small, reviewable summaries.

  launch list : ncu --metrics gpu__time_duration.sum --clock-control none -c N --csv --log-file ncu_out/L.csv <cmd>
                python scripts/ncu_summary.py launches ncu_out/L.csv ncu_out/<tag>_launch_list_summary.csv "<cmd>"
  full set    : ncu --set full --clock-control none --import-source on -k regex:... -o ncu_out/R <cmd>
                ncu -i ncu_out/R.ncu-rep --page raw --csv > ncu_out/R_raw.csv
                python scripts/ncu_summary.py full ncu_out/R_raw.csv ncu_out/<tag>_ncu_full_summary.json "<cmd>"

Numbers printed by the profiled command itself are never bench values.
"""
import collections
import csv
import io
import json
import sys

FULL_KEYS = [
    "Kernel Name", "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
    "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_dynamic",
    "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_registers", "smsp__inst_executed.sum",
    "lts__t_sector_hit_rate.pct", "lts__t_sectors_srcunit_tex_op_red.sum", "sm__cycles_elapsed.max",
    "smsp__thread_inst_executed_per_inst_executed.ratio",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_tensor.sum",
    "sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_uniform.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
    "lts__t_bytes.sum", "lts__t_sectors_srcunit_tex_op_read.sum", "nvlrx__bytes.sum", "nvltx__bytes.sum",
]
STALL_PREFIX = "smsp__average_warps_issue_stalled_"


def _rows(path):
    with open(path) as f:
        lines = [l for l in f if not l.startswith("==")]
    return list(csv.reader(io.StringIO("".join(lines))))


def launches(src, dst, cmd):
    rows = _rows(src)
    hdr = rows[0]
    ix = {k: hdr.index(k) for k in ("Kernel Name", "Metric Name", "Metric Unit", "Metric Value")}
    scale = {"ns": 1e-3, "nsecond": 1e-3, "us": 1.0, "usecond": 1.0, "ms": 1e3, "msecond": 1e3, "s": 1e6, "second": 1e6}
    agg = collections.OrderedDict()
    for r in rows[1:]:
        if len(r) <= ix["Metric Value"] or r[ix["Metric Name"]] != "gpu__time_duration.sum":
            continue
        us = float(r[ix["Metric Value"]].replace(",", "")) * scale.get(r[ix["Metric Unit"]], 1.0)
        a = agg.setdefault(r[ix["Kernel Name"]][:80], [0, 0.0])
        a[0] += 1
        a[1] += us
    total = sum(a[1] for a in agg.values()) or 1.0
    with open(dst, "w") as f:
        f.write("# %s\nkernel,launches,avg_us,share_of_listed_time\n" % cmd)
        for k, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write('"%s",%d,%.2f,%.4f\n' % (k, n, t / n, t / total))
    return agg


def full(src, dst, cmd):
    rows = _rows(src)
    hdr, units, data = rows[0], rows[1], rows[2:]
    keys = FULL_KEYS + [h for h in hdr if h.startswith(STALL_PREFIX) and h.endswith("_per_issue_active.ratio")]
    out = {"source": cmd, "launches": []}
    for r in data:
        d = {}
        for k in keys:
            if k in hdr:
                i = hdr.index(k)
                d[k] = (r[i] + " " + units[i]).strip()
        out["launches"].append(d)
    with open(dst, "w") as f:
        json.dump(out, f, indent=1)
    return out


if __name__ == "__main__":
    if len(sys.argv) < 4 or sys.argv[1] not in ("launches", "full"):
        sys.exit(__doc__)
    mode, src, dst = sys.argv[1:4]
    cmd = sys.argv[4] if len(sys.argv) > 4 else ""
    (launches if mode == "launches" else full)(src, dst, cmd)
    print("wrote", dst)
