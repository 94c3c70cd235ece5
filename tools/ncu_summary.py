"""Summarise Nsight Compute CSV exports into markdown: per-launch table, kernel shares, dram traffic per launch.
    python tools/ncu_summary.py launches launches_yolov5s.csv launches_yolov5s.md
    python tools/ncu_summary.py metrics  conv_metrics_yolov5s.csv conv_metrics_yolov5s.md yolov5s
The metrics mode also records the per-model dram traffic in profiles/traffic.json (read by bench.py's roofline record)."""
import collections
import csv
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def read(path):
    lines = [l for l in open(path) if not l.startswith("==")]
    return list(csv.DictReader(lines))


def to_us(v, unit):
    v = float(v.replace(",", ""))
    return {"ns": v / 1e3, "us": v, "ms": v * 1e3, "s": v * 1e6}.get(unit, v)


def to_bytes(v, unit):
    v = float(v.replace(",", ""))
    return v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1)


def short(name):
    n = name.replace("void ", "").replace("y5::", "")
    return n.split("(")[0][:60]


def launches(src, dst):
    rows = read(src)
    agg = collections.OrderedDict()
    for r in rows:
        if r["Metric Name"] != "gpu__time_duration.sum":
            continue
        agg.setdefault(short(r["Kernel Name"]), []).append(to_us(r["Metric Value"], r["Metric Unit"]))
    tot = sum(sum(v) for v in agg.values())
    with open(dst, "w") as f:
        f.write(f"# ncu launch list ({os.path.basename(src)}): gpu__time_duration.sum, --clock-control none\n\n")
        f.write("Per-launch times under ncu are cold-cache and serialised: compare SHARES, not absolutes.\n\n")
        f.write("| kernel | launches | total us | share | avg us | max us |\n|---|---:|---:|---:|---:|---:|\n")
        for k, v in sorted(agg.items(), key=lambda kv: -sum(kv[1])):
            f.write(f"| `{k}` | {len(v)} | {sum(v):.1f} | {100 * sum(v) / tot:.1f}% | {sum(v) / len(v):.1f} | {max(v):.1f} |\n")
        f.write(f"\ntotal {tot:.1f} us over {sum(len(v) for v in agg.values())} launches\n")
    print(open(dst).read())


def metrics(src, dst, workload):
    rows = read(src)
    per = collections.OrderedDict()
    for r in rows:
        per.setdefault(r["ID"], {"name": short(r["Kernel Name"]), "grid": r.get("Grid Size", "")})[r["Metric Name"]] = (r["Metric Value"], r["Metric Unit"])
    n, dram, l2, dur = 0, 0.0, 0.0, 0.0
    with open(dst, "w") as f:
        f.write(f"# ncu per-launch metrics of conv_gemm_kernel ({os.path.basename(src)})\n\n")
        f.write("| # | kernel | grid | us | dram R MB | dram W MB | L2 MB | tensor pipe % | SM % |\n|---|---|---|---:|---:|---:|---:|---:|---:|\n")
        for i, m in per.items():
            g = lambda k: m.get(k, ("0", ""))  # noqa: E731
            us = to_us(*g("gpu__time_duration.sum"))
            r, w = to_bytes(*g("dram__bytes_read.sum")), to_bytes(*g("dram__bytes_write.sum"))
            l = to_bytes(*g("lts__t_bytes.sum"))
            tp = float(g("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active")[0].replace(",", ""))
            sm = float(g("sm__throughput.avg.pct_of_peak_sustained_elapsed")[0].replace(",", ""))
            f.write(f"| {i} | `{m['name']}` | {m['grid']} | {us:.1f} | {r / 1e6:.1f} | {w / 1e6:.1f} | {l / 1e6:.1f} | {tp:.1f} | {sm:.1f} |\n")
            n += 1; dram += r + w; l2 += l; dur += us
        f.write(f"\n{n} launches, {dur:.1f} us, DRAM traffic {dram / 1e6:.1f} MB ({dram / n / 1e6:.2f} MB per launch), L2 traffic {l2 / 1e6:.1f} MB\n")
    tj = os.path.join(ROOT, "profiles", "traffic.json")
    os.makedirs(os.path.dirname(tj), exist_ok=True)
    t = json.load(open(tj)) if os.path.exists(tj) else {}
    t[workload] = dram / n
    t[workload + "_l2_bytes_per_launch"] = l2 / n
    json.dump(t, open(tj, "w"), indent=1)
    print(open(dst).read()[-600:])


def launches_bw(src, dst, title="training step"):
    """launch list with DRAM bytes: per kernel launches / time / share and the DRAM bandwidth it ran at (cold caches under ncu)."""
    rows = read(src)
    per = collections.OrderedDict()
    for r in rows:
        per.setdefault(r["ID"], {"name": short(r["Kernel Name"])})[r["Metric Name"]] = (r["Metric Value"], r["Metric Unit"])
    agg = collections.OrderedDict()
    for m in per.values():
        g = lambda k: m.get(k, ("0", ""))  # noqa: E731
        a = agg.setdefault(m["name"], [0, 0.0, 0.0, 0.0, 0.0])
        us = to_us(*g("gpu__time_duration.sum"))
        a[0] += 1
        a[1] += us
        a[2] += to_bytes(*g("dram__bytes_read.sum"))
        a[3] += to_bytes(*g("dram__bytes_write.sum"))
        a[4] = max(a[4], us)
    tot = sum(a[1] for a in agg.values())
    with open(dst, "w") as f:
        f.write(f"# ncu launch list of one {title} ({os.path.basename(src)}): gpu__time_duration.sum + dram bytes, --clock-control none\n\n")
        f.write("Per-launch times under ncu are cold-cache and serialised: compare SHARES, not absolutes.\n\n")
        f.write("| kernel | launches | total us | share | avg us | max us | DRAM read MB | DRAM write MB | DRAM GB/s |\n|---|---:|---:|---:|---:|---:|---:|---:|---:|\n")
        for k, a in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write(f"| `{k}` | {a[0]} | {a[1]:.1f} | {100 * a[1] / tot:.1f}% | {a[1] / a[0]:.1f} | {a[4]:.1f} | {a[2] / 1e6:.1f} | {a[3] / 1e6:.1f} | "
                    f"{(a[2] + a[3]) / a[1] / 1e3:.0f} |\n")
        f.write(f"\ntotal {tot:.1f} us over {sum(a[0] for a in agg.values())} launches, DRAM traffic "
                f"{sum(a[2] + a[3] for a in agg.values()) / 1e9:.2f} GB\n")
    print(open(dst).read())


if __name__ == "__main__":
    {"launches": launches, "metrics": metrics, "launches_bw": launches_bw}[sys.argv[1]](*sys.argv[2:])
