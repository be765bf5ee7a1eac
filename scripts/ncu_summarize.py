"""Summarise an `ncu --csv --metrics ...` per-launch log (one row per launch and metric) per kernel family:
launches, total / share of the device time, DRAM bytes and achieved GB/s, tensor-pipe and issue-slot utilisation.
Optionally writes profiles/r2_traffic.json (DRAM bytes per launch of the dominant kernels, read by bench.py).

    python scripts/ncu_summarize.py <run>/all_kernels.csv [--traffic profiles/r2_traffic.json]
    python scripts/ncu_summarize.py <run>/kpconv_op.csv --op kpconv_32_32 --iters 3 --traffic profiles/r2_traffic.json

The second form is for a log of ONE operator repeated `--iters` times (scripts/ncu_targets.py with ONLY=kpconv): the
DRAM bytes of every launch are summed and divided by the repetitions, and stored under the key bench.py looks up
(`kpconv_<Cin>_<Cout>`: all kernels of one d3f_kpconv_forward call), merged into an existing traffic file.
"""
import collections
import csv
import json
import re
import sys


def main():
    path = sys.argv[1]
    traffic_out = sys.argv[sys.argv.index("--traffic") + 1] if "--traffic" in sys.argv else None
    if traffic_out:
        os.makedirs(os.path.dirname(os.path.abspath(traffic_out)), exist_ok=True)
    rows = [r for r in csv.reader(open(path, errors="replace")) if len(r) > 10]
    hdr = rows[0]
    ik, im, iv, iu, iid = hdr.index("Kernel Name"), hdr.index("Metric Name"), hdr.index("Metric Value"), \
        hdr.index("Metric Unit"), hdr.index("ID")
    launches = collections.OrderedDict()
    for r in rows[1:]:
        d = launches.setdefault(r[iid], {"name": r[ik]})
        try:
            v = float(r[iv].replace(",", ""))
        except ValueError:
            continue
        u = r[iu]
        scale = {"Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "byte": 1.0, "us": 1e-6, "ms": 1e-3, "ns": 1e-9, "s": 1.0,
                 "usecond": 1e-6, "msecond": 1e-3, "nsecond": 1e-9, "second": 1.0}.get(u, 1.0)
        d[r[im]] = v * scale
    fam = collections.OrderedDict()
    for d in launches.values():
        name = re.sub(r"\(.*", "", d["name"].replace("(int)", "").replace("(bool)", "")).replace("void ", "").replace("d3f::", "").replace("(anonymous namespace)::", "")
        f = fam.setdefault(name, collections.defaultdict(float))
        f["n"] += 1
        f["t"] += d.get("gpu__time_duration.sum", 0.0)
        f["rd"] += d.get("dram__bytes_read.sum", 0.0)
        f["wr"] += d.get("dram__bytes_write.sum", 0.0)
        w = d.get("gpu__time_duration.sum", 0.0)
        for k, m in (("tensor", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"),
                     ("issue", "smsp__issue_active.avg.pct_of_peak_sustained_active"),
                     ("warps", "sm__warps_active.avg.pct_of_peak_sustained_active"),
                     ("l2hit", "lts__t_sector_hit_rate.pct"),
                     ("l2bytes", "lts__t_bytes.sum")):
            if k == "l2bytes":
                f[k] += d.get(m, 0.0)
            else:
                f[k] += d.get(m, 0.0) * w      # time-weighted
    total = sum(f["t"] for f in fam.values())
    print("# per-kernel counters of one step (ncu, cold caches between launches: compare SHARES, not absolutes)")
    print("# total device time of the %d launches: %.1f us" % (len(launches), total * 1e6))
    print("%-46s %4s %9s %6s %9s %9s %8s %7s %7s %7s %6s" % ("kernel", "n", "time us", "share", "DRAM MB", "DRAM GB/s", "L2 GB/s",
                                                             "tensor%", "issue%", "warps%", "L2hit%"))
    traffic = {}
    for name, f in sorted(fam.items(), key=lambda kv: -kv[1]["t"]):
        t = f["t"] or 1e-30
        print("%-46s %4d %9.1f %5.1f%% %9.2f %9.0f %8.0f %7.1f %7.1f %7.1f %6.1f" % (
            name[:46], f["n"], t * 1e6, 100 * t / total, (f["rd"] + f["wr"]) / 1e6, (f["rd"] + f["wr"]) / t / 1e9,
            f["l2bytes"] / t / 1e9, f["tensor"] / t, f["issue"] / t, f["warps"] / t, f["l2hit"] / t))
        traffic[name] = dict(dram_bytes_per_launch=(f["rd"] + f["wr"]) / f["n"], launches=int(f["n"]),
                             source="ncu dram__bytes_read.sum + dram__bytes_write.sum, " + path)
    if "--op" in sys.argv:
        import os
        key = sys.argv[sys.argv.index("--op") + 1]
        iters = int(sys.argv[sys.argv.index("--iters") + 1]) if "--iters" in sys.argv else 1
        tot = sum(f["rd"] + f["wr"] for f in fam.values()) / iters
        n = sum(f["n"] for f in fam.values()) / iters
        print("# %s: %.2f MB of DRAM traffic per call over %.1f launches" % (key, tot / 1e6, n))
        traffic = json.load(open(traffic_out)) if traffic_out and os.path.exists(traffic_out) else {}
        traffic[key] = dict(dram_bytes_per_launch=tot, launches=n,
                            source="ncu dram__bytes_read.sum + dram__bytes_write.sum over every kernel of one call, " + path)
    if traffic_out:
        json.dump(traffic, open(traffic_out, "w"), indent=1)


if __name__ == "__main__":
    main()
