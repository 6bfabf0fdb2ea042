#!/usr/bin/env python
"""Eager-PyTorch training baseline on one GPU (informative, beside scripts/train_bench.py): the oracle restatement's
p_losses (oracle/restatement.py) and its backward at BASELINE config 5's shape, as the reference trains — fp16 autocast
with a GradScaler, torch.utils.checkpoint around every ResBlock and SpatialTransformer (the yaml's use_checkpoint),
`F.scaled_dot_product_attention` for the attention, cuDNN / cuBLAS for everything else — the appearance net and the
pose ControlNet trained by AdamW (lr 1e-5), the SD UNet frozen.

A measurement helper under tests/ like tests/torch_gpu_baseline.py (only tests/ may execute oracle/), not a pytest
module; nothing in the product imports it.

    python tests/torch_gpu_train_baseline.py [--batch 4] [--latent 64] [--steps 5] [--warmup 2]

Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from scripts.train_bench import REFERENCE_GF_PER_SAMPLE, gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--latent", type=int, default=64)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    from torch.utils.checkpoint import checkpoint
    from magicdance_b200 import synth
    from oracle import restatement as R

    assert torch.cuda.is_available(), "needs a GPU"
    torch.backends.cuda.matmul.allow_tf32 = True  # train_tiktok.py's defaults for the conv / matmul libraries
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cudnn.benchmark = True

    def sdpa_attention(sd, p, x, context, heads):
        q, k, v = R._lin(sd, p + "to_q", x), R._lin(sd, p + "to_k", context), R._lin(sd, p + "to_v", context)
        b, n, c = q.shape
        q, k, v = (t.reshape(b, -1, heads, c // heads).transpose(1, 2) for t in (q, k, v))
        return R._lin(sd, p + "to_out.0", F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(b, n, c))

    R.attention = sdpa_attention
    resblock, transformer = R.resblock, R.spatial_transformer
    R.resblock = lambda *a: checkpoint(resblock, *a, use_reentrant=False)
    R.spatial_transformer = lambda *a: checkpoint(transformer, *a, use_reentrant=False)

    sd = synth.synth_state_dict(seed=0, device="cuda")
    trained = [v.requires_grad_() for k, v in sd.items() if k.startswith((R.APPEARANCE, R.POSE))]
    opt = torch.optim.AdamW(trained, lr=1e-5)
    scaler = torch.amp.GradScaler("cuda")
    B, L = args.batch, args.latent
    inp = {k: v.cuda() for k, v in synth.synth_inputs(B, L, seed=0, shared_reference=False).items()}
    g = torch.Generator(device="cuda").manual_seed(0)
    x0 = 0.9 * torch.randn(B, 4, L, L, device="cuda", generator=g)

    def step():
        t = torch.randint(0, 1000, (B,), device="cuda", generator=g)
        noise = torch.randn(x0.shape, device="cuda", generator=g)
        with torch.autocast("cuda", dtype=torch.float16):
            loss, _, _ = R.p_losses(sd, x0, t, noise, inp["context"], inp["pose"], inp["ref"])
        scaler.scale(loss).backward()
        scaler.step(opt)
        scaler.update()
        opt.zero_grad(set_to_none=True)
        return loss

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(args.steps):
        loss = step()
    end.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(end) / args.steps
    name, limit = gpu_info()
    print(json.dumps({
        "impl": "torch-eager-gpu training (oracle restatement, fp16 autocast + GradScaler, torch.utils.checkpoint, "
                "SDPA, cuDNN/cuBLAS)",
        "metric": "training samples/s (BASELINE config 5, stage 2, one GPU)", "device": name, "power_limit_w": limit,
        "batch": B, "latent": L, "steps": args.steps, "warmup": args.warmup, "samples_per_s": B * 1e3 / ms,
        "ms_per_step": ms, "peak_allocated_gib": torch.cuda.max_memory_allocated() / 2 ** 30,
        "algorithmic_tflops_vs_reference_count": REFERENCE_GF_PER_SAMPLE * B / ms, "finite": bool(torch.isfinite(loss))}))


if __name__ == "__main__":
    main()
