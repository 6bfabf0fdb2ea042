"""Condenses Nsight Compute outputs into small text summaries (profiles/ is where they go; git ignores them).

  python scripts/ncu_summary.py rep   prof.ncu-rep      > profiles/ncu_top_kernels.md
  python scripts/ncu_summary.py list  launches.csv      > profiles/launch_list_step.md
"""
import collections
import csv
import io
import re
import subprocess
import sys

KEYS = [
    ("gpu__time_duration.sum", "time"),
    ("l1tex__m_xbar2l1tex_read_bytes.sum", "l2->sm bytes"),
    ("lts__t_bytes.sum", "l2 bytes"),
    ("launch__waves_per_multiprocessor", "waves/SM"),
    ("launch__registers_per_thread", "regs"),
    ("dram__bytes_read.sum", "dram_rd"),
    ("dram__bytes_write.sum", "dram_wr"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram%"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor%"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm%"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps%"),
]


def rep(path):
    """path: a .ncu-rep, or the CSV `ncu -i x.ncu-rep --page raw --csv` printed (what travels back from the GPU box)"""
    if path.endswith(".csv"):
        raw = "".join(l for l in open(path) if not l.startswith("=="))
    else:
        raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    print(f"# ncu --set full --clock-control none: per-launch metrics ({path})\n")
    print("| kernel | grid | " + " | ".join(k for _, k in KEYS) + " |")
    print("|---|---|" + "---|" * len(KEYS))
    for r in data:
        name = r[hdr.index("Kernel Name")].split("(")[0].replace("void mdb::", "").replace("mdb::", "")
        cells = []
        for full, _ in KEYS:
            if full in hdr:
                i = hdr.index(full)
                v = r[i]
                try:
                    v = f"{float(v):.2f}"
                except ValueError:
                    pass
                cells.append(f"{v} {units[i]}".strip())
            else:
                cells.append("n/a")
        print(f"| {name} | {r[hdr.index('Grid Size')]} | " + " | ".join(cells) + " |")


def launch_list(path):
    with open(path) as f:
        lines = [l for l in f if not l.startswith("==")]
    rows = list(csv.DictReader(lines))
    # one row per (launch ID, metric): fold into launches
    launches, order = {}, []
    for r in rows:
        i = r["ID"]
        if i not in launches:
            launches[i] = {"name": r["Kernel Name"]}
            order.append(i)
        v = float(r["Metric Value"].replace(",", ""))
        unit = r["Metric Unit"]
        if r["Metric Name"] == "gpu__time_duration.sum":
            launches[i]["us"] = v / 1e3 if unit in ("ns", "nsecond") else (v * 1e3 if unit in ("ms", "msecond") else v)
        else:
            scale = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1.0)
            launches[i][r["Metric Name"]] = v * scale
    seq = [launches[i] for i in order]
    ends = [j for j, r in enumerate(seq) if "cfg_ddim_update" in r["name"]]
    step = seq[ends[-2] + 1: ends[-1] + 1] if len(ends) >= 2 else seq
    tot, cnt, rd, wr = collections.Counter(), collections.Counter(), collections.Counter(), collections.Counter()
    for r in step:
        nm = re.sub(r"\(.*", "", r["name"]).replace("void mdb::", "").replace("mdb::", "")
        tot[nm] += r.get("us", 0.0)
        cnt[nm] += 1
        rd[nm] += r.get("dram__bytes_read.sum", 0.0)
        wr[nm] += r.get("dram__bytes_write.sum", 0.0)
    total = sum(tot.values())
    print(f"# ncu launch list (gpu__time_duration.sum + DRAM bytes, --clock-control none; cold-cache and serialised:\n"
          f"# compare SHARES, not absolutes) — this library's kernels of ONE captured DDIM step ({path})\n")
    print(f"one step: {sum(cnt.values())} kernel launches, {total / 1e3:.2f} ms summed kernel time, "
          f"DRAM read {sum(rd.values()) / 1e9:.2f} GB, written {sum(wr.values()) / 1e9:.2f} GB\n")
    print("| kernel | launches | total us | share | avg us | DRAM read MB | DRAM written MB |")
    print("|---|---|---|---|---|---|---|")
    for k, v in tot.most_common():
        print(f"| {k[:80]} | {cnt[k]} | {v:.1f} | {100 * v / total:.1f}% | {v / cnt[k]:.2f} | {rd[k] / 1e6:.1f} | {wr[k] / 1e6:.1f} |")


if __name__ == "__main__":
    {"rep": rep, "list": launch_list}[sys.argv[1]](sys.argv[2])
