"""Condense `ncu -i <rep> --page raw --csv` into one line per kernel launch.

    ncu -i /tmp/profile_all.ncu-rep --page raw --csv > /tmp/raw.csv && python tools/ncu_summary.py /tmp/raw.csv
"""
import csv
import sys

WANT = [("gpu__time_duration.sum", "us", 1e-3), ("dram__bytes_read.sum", "dram_rd_MB", None), ("dram__bytes_write.sum", "dram_wr_MB", None),
        ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram%", 1), ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2%", 1),
        ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm%", 1),
        ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor%", 1),
        ("sm__ops_path_tensor_op_utchmma_src_tf32_dst_fp32_sparsity_off.avg.pct_of_peak_sustained_elapsed", "tf32op%", 1),
        ("l1tex__m_xbar2l1tex_read_bytes.sum", "xbar_rd_MB", None),
        ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps%", 1), ("launch__registers_per_thread", "regs", 1),
        ("lts__t_sector_hit_rate.pct", "L2hit%", 1)]


def to_bytes(v, unit):
    m = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
    return float(v) * m.get(unit, 1)


rows = list(csv.reader(open(sys.argv[1])))
hdr = next(i for i, r in enumerate(rows) if r and r[0] == "ID")
names, units = rows[hdr], rows[hdr + 1]
col = {n: i for i, n in enumerate(names)}
print("%-44s %-14s %9s %9s %9s %6s %6s %6s %8s %8s %9s %7s %5s %7s" % ("kernel", "grid", "us", "dram_rdMB", "dram_wrMB", "dram%", "L2%", "sm%", "tensor%", "tf32op%", "xbar_rdMB", "warps%", "regs", "L2hit%"))
agg = {}
for r in rows[hdr + 2:]:
    if len(r) < len(names):
        continue
    name = r[col["Kernel Name"]].split("(")[0][:44]
    grid = r[col["Grid Size"]].replace(" ", "") if "Grid Size" in col else ""
    vals = {}
    for key, label, scale in WANT:
        if key not in col or r[col[key]] in ("", "n/a"):
            vals[label] = float("nan")
            continue
        v = r[col[key]].replace(",", "")
        if label.endswith("_MB") or label.endswith("MB"):
            vals[label] = to_bytes(v, units[col[key]]) / 1e6
        elif label == "us":
            u = units[col[key]]
            vals[label] = float(v) * {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}.get(u, 1e-3)
        else:
            vals[label] = float(v)
    print("%-44s %-14s %9.2f %9.3f %9.3f %6.1f %6.1f %6.1f %8.2f %8.2f %9.3f %7.1f %5.0f %7.1f" % (name, grid, vals["us"], vals["dram_rd_MB"], vals["dram_wr_MB"],
          vals["dram%"], vals["L2%"], vals["sm%"], vals["tensor%"], vals["tf32op%"], vals["xbar_rd_MB"], vals["warps%"], vals["regs"], vals["L2hit%"]))
    a = agg.setdefault(name, [0, 0.0])
    a[0] += 1; a[1] += vals["us"]
print()
print("per-kernel totals (cold-cache, serialised ncu replays: compare shares, not absolutes)")
tot = sum(v[1] for v in agg.values())
for k, (n, us) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print("%-44s n=%4d  total %10.1f us  avg %9.2f us  share %5.1f%%" % (k, n, us, us / n, 100 * us / tot))
