"""Where the time of one denoising step goes, per launch, against what the hardware could do.

    python scripts/step_profile.py [--batch 1 8] [--tune k=v[,k=v]] [--tag name] [--out profiles]

Builds the pipeline bench.py measures (synthetic weights, 64x64 latent, pose ControlNet + the cond/uncond UNet pair),
then runs one eager `DenoisePipeline.step` under torch.profiler with CUDA activities.  The eager step issues every
kernel on one stream, so its GEMM / implicit-GEMM launches can be joined in launch order with the shapes `ops.TRACE`
records; inside the graph bench.py replays, the pose ControlNet and a few branches run on other streams and that order
is lost.  The kernels and their plans are the same in both.  The timestep MLPs run in the eager step but not in the graph
(they are tabulated once per schedule); they are listed under "other".

For every launch: kernel, grid, duration; for GEMM launches (m, n, k, conv, splits) and the bound
max(weight bytes / 3.35 TB/s, 2mnk / 989 TFLOP/s) (H100 SXM data sheet: HBM3 bandwidth, dense FP16).  The gap
(duration - bound) is summed by class.  A GEMM is "deep" when its rows are the tokens of the 16x16 level or a deeper
one.  Writes <out>/step_profile_<tag>_B<batch>.md.  `--tune` sets ops.tuning keys for the whole run, so two plans can
be profiled in one process (e.g. `--tune skinny_ctas=0` for the compute-bound plan)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

HBM = 3.35e12
PEAK = 989e12
CHANNELS = (320, 640, 1280)
GEMM_KERNELS = ("gemm_tc_kernel", "gemm_igemm_kernel", "splitk_finalize_kernel")


def classify(name, shape, batch):
    if shape is not None:
        m, n, k, conv = shape[:4]
        tokens = n if (conv is None and m in CHANNELS and n not in CHANNELS) else m  # V^T GEMMs: M = channels
        return "deep GEMM/conv" if tokens <= 2 * batch * 256 else "other GEMM/conv"
    low = name.lower()
    if "attn" in low:
        return "attention"
    if any(s in low for s in ("gn_", "layernorm", "groupnorm")):
        return "norm"
    return "elementwise/other"


def profile(batch, latent, tune):
    import torch
    from magicdance_b200 import ops, synth
    from magicdance_b200.engine import DenoiseEngine
    from magicdance_b200.pipeline import DenoisePipeline
    from torch.profiler import ProfilerActivity, profile as tprofile

    torch.set_grad_enabled(False)
    dev = "cuda:0"
    eng = DenoiseEngine(synth.synth_state_dict(seed=0, device=dev), device=dev)
    pipe = DenoisePipeline(eng, ddim_steps=50, scale=7.0, eta=0.0)
    inp = synth.synth_inputs(batch, latent, seed=100, shared_reference=True)
    x = inp["x"][:1].expand(batch, -1, -1, -1).contiguous().to(dev)
    ctx = inp["context"][:1].to(dev)
    with ops.tuning(**tune):
        hint = pipe.hint(inp["pose"].to(dev))
        bank = pipe.reference_bank(inp["ref"][:1].to(dev), ctx, 49, first_only=True)
        for _ in range(2):  # warm: modules, tensor maps, the text K/V cache
            pipe.step(x, 49, ctx, hint, bank)
        torch.cuda.synchronize()
        ops.TRACE = []
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            pipe.step(x, 49, ctx, hint, bank)
            torch.cuda.synchronize()
        trace, ops.TRACE = ops.TRACE, None
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "t.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    kernels = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    rows, gi = [], 0
    for e in kernels:
        name = e["name"]
        shape = None
        if any(g in name for g in GEMM_KERNELS[:2]):
            assert gi < len(trace), "more GEMM launches than ops.TRACE entries"
            shape = trace[gi]
            gi += 1
        elif GEMM_KERNELS[2] in name:
            shape = rows[-1]["shape"]  # the second pass of the GEMM before it (explicit split counts above 8)
        dur = float(e["dur"])
        bound = 0.0
        if shape is not None and GEMM_KERNELS[2] not in name:
            m, n, k = shape[:3]
            bound = max(2.0 * n * k / HBM, 2.0 * m * n * k / PEAK) * 1e6
        rows.append(dict(name=name, grid=e.get("args", {}).get("grid"), dur=dur, shape=shape, bound=bound,
                         cls=classify(name, shape, batch)))
    assert gi == len(trace), f"{len(trace)} GEMM calls traced, {gi} GEMM kernels profiled"
    return rows


def short(name):
    name = name.replace("void ", "").replace("mdb::", "")
    return name if len(name) <= 60 else name[:57] + "..."


def write(rows, batch, tag, out, gpu):
    os.makedirs(out, exist_ok=True)
    path = os.path.join(out, f"step_profile_{tag}_B{batch}.md")
    classes = ("deep GEMM/conv", "other GEMM/conv", "attention", "norm", "elementwise/other")
    tot = {c: [0, 0.0, 0.0] for c in classes}
    for r in rows:
        t = tot[r["cls"]]
        t[0] += 1
        t[1] += r["dur"]
        t[2] += r["bound"]
    lines = [f"# One eager denoising step, {batch} frame(s) at a 64x64 latent — {tag}", "", f"GPU: {gpu}", "",
             "| class | launches | time µs | bound µs | gap µs |", "|---|---|---|---|---|"]
    for c in classes:
        n_, d_, b_ = tot[c]
        lines.append(f"| {c} | {n_} | {d_:.1f} | {b_:.1f} | {d_ - b_:.1f} |")
    s = sum(r["dur"] for r in rows)
    lines += [f"| total | {len(rows)} | {s:.1f} | | |", "", "| # | kernel | grid | µs | m, n, k, conv, splits | bound µs | class |",
              "|---|---|---|---|---|---|---|"]
    for i, r in enumerate(rows):
        sh = r["shape"]
        shs = "" if sh is None else f"{sh[0]}, {sh[1]}, {sh[2]}, {sh[3]}, {sh[5]}"
        lines.append(f"| {i} | `{short(r['name'])}` | {r['grid']} | {r['dur']:.1f} | {shs} | {r['bound']:.1f} | {r['cls']} |")
    with open(path, "w") as f:
        f.write("\n".join(lines) + "\n")
    print("\n".join(lines[:13]), flush=True)
    print(f"wrote {path}", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--latent", type=int, default=64)
    ap.add_argument("--tune", default="", help="ops.tuning keys as k=v[,k=v]")
    ap.add_argument("--tag", default="default")
    ap.add_argument("--out", default=os.path.join(REPO, "profiles"))
    args = ap.parse_args()
    tune = {k: int(v) for k, v in (kv.split("=") for kv in args.tune.split(",") if kv)}
    import torch
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    gpu = f"{torch.cuda.get_device_name()} | nvidia-smi: {smi}"
    for b in args.batch:
        write(profile(b, args.latent, tune), b, args.tag, args.out, gpu)


if __name__ == "__main__":
    main()
