"""Turn ncu exports into small JSON summaries.

  python tools/ncu_summary.py kernel <raw.csv from `ncu -i X.ncu-rep --page raw --csv`> <out.json> "<what>"
  python tools/ncu_summary.py launches <launch list csv from `ncu --metrics gpu__time_duration.sum --csv --log-file`> <out.json> "<what>"
"""
import collections
import csv
import json
import sys

KEEP = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        "l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "launch__shared_mem_config_size",
        "launch__occupancy_limit_shared_mem", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct", "smsp__inst_executed.sum",
        "smsp__thread_inst_executed_per_inst_executed.ratio", "l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio"]


def kernel(path, out, what):
    rows = list(csv.reader(open(path)))
    hdr, units = rows[0], rows[1]
    launches = []
    for vals in rows[2:]:
        d = dict(zip(hdr, vals))
        u = dict(zip(hdr, units))
        rec = {"Kernel Name": d.get("Kernel Name", "")}
        for k in KEEP:
            if k in d and d[k] != "":
                rec[k] = ("%s %s" % (d[k], u.get(k, ""))).strip()
        launches.append(rec)
    json.dump({"what": what, "launches": launches}, open(out, "w"), indent=1)


def launches(path, out, what):
    rows = list(csv.reader(open(path)))
    hi = [i for i, r in enumerate(rows) if r and r[0] == "ID"][0]
    hdr = rows[hi]
    ki, vi = hdr.index("Kernel Name"), hdr.index("Metric Value")
    agg = collections.OrderedDict()
    for r in rows[hi + 1:]:
        if len(r) <= vi:
            continue
        a = agg.setdefault(r[ki][:90], [0, 0.0])
        a[0] += 1
        a[1] += float(r[vi].replace(",", "")) / 1000.0
    tot = sum(v[1] for v in agg.values())
    ks = [{"kernel": k, "launches": v[0], "total_us": round(v[1], 1), "share_pct": round(100 * v[1] / tot, 2),
           "avg_us": round(v[1] / v[0], 2)} for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1])]
    json.dump({"what": what, "kernels": ks}, open(out, "w"), indent=1)


if __name__ == "__main__":
    {"kernel": kernel, "launches": launches}[sys.argv[1]](sys.argv[2], sys.argv[3], sys.argv[4])
