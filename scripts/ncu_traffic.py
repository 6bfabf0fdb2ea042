"""profiles/traffic.json from the ncu launch lists of one captured DDIM step (NVTX-scoped: `bench.py --nvtx` under
`ncu --nvtx --nvtx-include "mdb_step/"` with dram__bytes_read.sum / dram__bytes_write.sum / gpu__time_duration.sum):
per frames-per-GPU, the DRAM bytes and time of the wgmma GEMM (gemm_tc_kernel) and of attention.

    python scripts/ncu_traffic.py profiles/traffic.json 1=gpurun_out/launches_b1.csv 8=gpurun_out/launches_b8.csv
"""
import collections
import csv
import json
import sys


def one(path, frames):
    rows = list(csv.DictReader(l for l in open(path) if not l.startswith("==")))
    by_id = collections.OrderedDict()
    for r in rows:
        d = by_id.setdefault(r["ID"], {"name": r["Kernel Name"]})
        v = float(r["Metric Value"].replace(",", ""))
        u = r["Metric Unit"]
        scale = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1e-9, "nsecond": 1e-9, "us": 1e-6, "usecond": 1e-6,
                 "ms": 1e-3, "msecond": 1e-3, "s": 1, "second": 1}.get(u, 1)
        d[r["Metric Name"]] = v * scale
    launches = list(by_id.values())
    ends = [i for i, l in enumerate(launches) if "cfg_ddim_update" in l["name"]]
    step = launches[ends[-2] + 1: ends[-1] + 1] if len(ends) >= 2 else launches
    out = {}
    for key, pats in (("gemm_tc_kernel_b%d" % frames, ("gemm_tc_kernel",)), ("attention_b%d" % frames, ("attn",))):
        sel = [l for l in step if any(p in l["name"] for p in pats)]
        rd = sum(l.get("dram__bytes_read.sum", 0) for l in sel)
        wr = sum(l.get("dram__bytes_write.sum", 0) for l in sel)
        t = sum(l.get("gpu__time_duration.sum", 0) for l in sel)
        out[key] = {"frames_per_gpu": frames, "launches_per_step": len(sel), "dram_read_bytes_per_step": rd,
                    "dram_write_bytes_per_step": wr, "dram_bytes_per_launch_avg": (rd + wr) / max(len(sel), 1),
                    "kernel_seconds_per_step_ncu": t,
                    "source": "ncu --nvtx --nvtx-include mdb_step/ --metrics gpu__time_duration.sum,dram__bytes_read.sum,"
                              "dram__bytes_write.sum --clock-control none on `bench.py --nvtx --steps 3 --warmup 1`: ONE "
                              "replayed step graph (%s)" % path}
    return out


if __name__ == "__main__":
    res = {}
    for arg in sys.argv[2:]:
        frames, path = arg.split("=", 1)
        res.update(one(path, int(frames)))
    json.dump(res, open(sys.argv[1], "w"), indent=1)
    print(json.dumps({k: {kk: vv for kk, vv in v.items() if kk != "source"} for k, v in res.items()}, indent=1))
