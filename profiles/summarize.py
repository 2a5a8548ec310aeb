"""Turn raw profiler outputs (Nsight Compute CSV / reports) into markdown summaries.

    python profiles/summarize.py launches <launches.csv> <out.md>
    python profiles/summarize.py full <report.ncu-rep> <out.md>
"""
import collections
import csv
import io
import json
import re
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "dram__throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        "l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
        "sass__inst_executed_local_loads", "smsp__issue_active.avg.pct_of_peak_sustained_active"]


def short(name):
    return re.sub(r"\(.*", "", name).replace("dirb200::", "").replace("void ", "")


def launches(src, dst):
    lines = [l for l in open(src) if not l.startswith("==")]
    recs = collections.OrderedDict()
    for r in csv.DictReader(lines):
        d = recs.setdefault(r["ID"], {"name": short(r["Kernel Name"]), "grid": r["Grid Size"]})
        d[r["Metric Name"]] = (float(r["Metric Value"].replace(",", "")), r["Metric Unit"])
    rows = list(recs.values())
    us = lambda d: d["gpu__time_duration.sum"][0] / (1000 if d["gpu__time_duration.sum"][1].startswith("n") else 1)
    def mb(d, k):
        if k not in d:
            return 0.0
        v, u = d[k]
        return v * {"byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1, "Gbyte": 1e3}[u]
    note = None
    idx = [i for i, r in enumerate(rows) if r["name"] == "adam_kernel"]
    pidx = [i for i, r in enumerate(rows) if r["name"].startswith("prep_weights_all_kernel")]
    if len(idx) > 1:                       # one step = (adam, next adam]
        step = rows[idx[0] + 1:idx[1] + 1]
    elif len(pidx) > 1:                    # short capture: one step = [weight prep, next weight prep)
        step = rows[pidx[0]:pidx[1]]
        note = ("NOTE: the capture held one complete step only, the FIRST step after the model was built -- it carries "
                "~160 one-time `FillFunctor` launches (lazily created gradient views); a steady-state step has 538 "
                "launches (bench.py `gpu_launches_per_step`).  The conv / BN launches are those of every step.")
    else:
        step = rows
    tot = collections.defaultdict(lambda: [0, 0.0, 0.0])
    for d in step:
        a = tot[d["name"]]
        a[0] += 1
        a[1] += us(d)
        a[2] += mb(d, "dram__bytes_read.sum") + mb(d, "dram__bytes_write.sum")
    total = sum(a[1] for a in tot.values())
    out = [f"# ncu launch list of ONE training step ({len(step)} launches, batch 256)", "",
           f"source: `{src}` (`ncu --metrics gpu__time_duration.sum[,dram__bytes_*] --clock-control none`; "
           "per-launch times are cold-cache and serialised: compare SHARES)", ""] + ([note, ""] if note else []) + [
           "| kernel | launches | ms | share | DRAM GB |", "|---|---:|---:|---:|---:|"]
    for k, a in sorted(tot.items(), key=lambda kv: -kv[1][1]):
        out.append(f"| `{k}` | {a[0]} | {a[1] / 1000:.3f} | {100 * a[1] / total:.1f}% | {a[2] / 1000:.2f} |")
    out.append(f"| **total** | {len(step)} | {total / 1000:.3f} | 100% | {sum(a[2] for a in tot.values()) / 1000:.2f} |")
    conv = [d for d in step if d["name"].startswith("igemm")]
    summary = {"conv_launches": len(conv), "conv_ms": sum(us(d) for d in conv) / 1000,
               "conv_dram_gb": sum(mb(d, "dram__bytes_read.sum") + mb(d, "dram__bytes_write.sum") for d in conv) / 1000}
    out += ["", f"conv kernels (igemm_kernel*): {json.dumps(summary)}"]
    open(dst, "w").write("\n".join(out) + "\n")
    json.dump(summary, open(dst.replace(".md", ".json"), "w"))
    print("\n".join(out[:14]))


def full(src, dst):
    raw = subprocess.run(["ncu", "-i", src, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    cols = [(k, hdr.index(k)) for k in KEYS if k in hdr]
    out = [f"# ncu --set full: {src}", "", "| # | kernel | grid | " + " | ".join(k for k, _ in cols) + " |",
           "|---|---|---|" + "---:|" * len(cols)]
    for n, r in enumerate(rows[2:]):
        out.append(f"| {n} | `{short(r[hdr.index('Kernel Name')])}` | {r[hdr.index('Grid Size')]} | " +
                   " | ".join(f"{float(r[i]):.4g}" if r[i] else "" for _, i in cols) + " |")
    out += ["", "units: " + ", ".join(f"{k}: {units[i]}" for k, i in cols)]
    open(dst, "w").write("\n".join(out) + "\n")
    print(f"{len(rows) - 2} kernels -> {dst}")


if __name__ == "__main__":
    {"launches": launches, "full": full}[sys.argv[1]](sys.argv[2], sys.argv[3])
