#!/usr/bin/env python
"""Secondary GPU baseline (BASELINE.md section 3, informative): the reference's path as plain eager PyTorch on
one H100 — the oracle restatement (oracle/restatement.py, the same functions the CPU baseline times) moved to
the GPU and run under fp16 autocast with cuDNN / cuBLAS, `F.scaled_dot_product_attention` standing in for the
xformers call the reference makes on a GPU (attention.py:242).  This is "the reference on this box": the number
the hand-written kernels have to beat, reported next to bench.py's line, never mixed into it.

It lives under tests/ because only tests/, smoke() and bench.py's CPU-baseline leg may execute oracle/; it is a
measurement helper, not a pytest module (no test_ prefix), and nothing in the product imports it.

    python tests/torch_gpu_baseline.py [--batch 1] [--steps 10] [--warmup 2] [--algorithmic]

default: one step = what the reference runs (appearance pass + pose + UNet-read, then pose again
+ UNet-uncond: 3124.4 GFLOP per frame-step).  --algorithmic: the bank is built once outside the timed region and
the discarded pose pass is skipped (2037.9 GFLOP), i.e. the same work bench.py's steady_state line counts.
Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", default="1", help="frames per step; a comma list runs several in one process")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--latent", type=int, default=64)
    ap.add_argument("--algorithmic", action="store_true")
    ap.add_argument("--no-sdpa", action="store_true", help="keep the vanilla einsum/softmax attention (attention.py:168-199)")
    ap.add_argument("--dtype", default="float16", choices=["float16", "bfloat16", "float32"])
    ap.add_argument("--device", default="cuda:0", help="cpu only to dry-run the script's logic at a tiny --latent")
    args = ap.parse_args()

    import numpy as np
    import torch
    import torch.nn.functional as F
    from magicdance_b200 import synth
    from oracle import restatement as R

    import time
    dev = args.device
    on_gpu = dev.startswith("cuda")
    assert not on_gpu or torch.cuda.is_available(), "needs a GPU (or --device cpu for a dry run)"
    torch.set_grad_enabled(False)
    torch.backends.cuda.matmul.allow_tf32 = True   # test_tiktok.py:358-359
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cudnn.benchmark = True

    if not args.no_sdpa:
        def sdpa_attention(sd, p, x, context, heads):
            q = R._lin(sd, p + "to_q", x)
            k = R._lin(sd, p + "to_k", context)
            v = R._lin(sd, p + "to_v", context)
            b, n, c = q.shape
            d = c // heads
            q, k, v = (t.reshape(b, -1, heads, d).transpose(1, 2) for t in (q, k, v))
            out = F.scaled_dot_product_attention(q, k, v)           # scale d^-0.5, no mask, no dropout
            return R._lin(sd, p + "to_out.0", out.transpose(1, 2).reshape(b, n, c))
        R.attention = sdpa_attention

    sd = synth.synth_state_dict(seed=0, device=dev)
    L = args.latent
    sched = R.ddim_schedule(R.make_schedule()["alphas_cumprod"].astype(np.float32).astype(np.float64))
    dtype = getattr(torch, args.dtype)
    sync = torch.cuda.synchronize if on_gpu else (lambda: None)

    def one(B):
        inp = {k: v.to(dev) for k, v in synth.synth_inputs(B, L, seed=0, shared_reference=True).items()}
        ctx = torch.autocast("cuda" if on_gpu else "cpu", dtype=dtype if on_gpu or dtype != torch.float16 else torch.bfloat16,
                             enabled=dtype != torch.float32)

        def step(x, index, bank_cache):
            t = torch.full((B,), int(sched["timesteps"][index]), dtype=torch.long, device=dev)
            if not args.algorithmic:
                x_prev, _, _, _ = R.p_sample_ddim(sd, x, t, index, inp["context"], inp["pose"], inp["ref"], sched, scale=7.0)
                return x_prev.float()
            bank = bank_cache[index]
            pose = R.controlnet_forward(sd, R.POSE, x, inp["pose"], t, inp["context"])
            e_c = R.unet_forward(sd, R.UNET, x, t, inp["context"], bank=bank, pose_control=pose, uc=False)
            e_u = R.unet_forward(sd, R.UNET, x, t, inp["context"], bank=[], pose_control=None, uc=True)
            e_t = e_u + 7.0 * (e_c - e_u)
            return R.ddim_update(x, e_t.float(), index, sched)[0].float()

        n = args.warmup + args.steps
        idxs = [49 - (i % 50) for i in range(n)]
        bank_cache = {}
        with ctx:
            if args.algorithmic:
                for ix in sorted(set(idxs)):
                    t = torch.full((B,), int(sched["timesteps"][ix]), dtype=torch.long, device=dev)
                    bank_cache[ix] = R.appearance_forward(sd, R.APPEARANCE, inp["ref"], t, inp["context"])
            x = inp["x"]
            t_start = 0.0
            for i, ix in enumerate(idxs):
                if i == args.warmup:
                    sync()
                    t_start = time.perf_counter()   # whole-chain wall clock between two device synchronisations
                x = step(x, ix, bank_cache)
            sync()
        sec = (time.perf_counter() - t_start) / args.steps
        gf = 2037.9 if args.algorithmic else 3124.4
        return {
            "impl": "torch-eager-gpu (oracle restatement under autocast; cuDNN/cuBLAS" + ("" if args.no_sdpa else "/SDPA") + ")",
            "metric": "denoise-steps/sec @512x512 50-step DDIM", "value": B / sec, "unit": "frame-steps/s",
            "ms_per_step": sec * 1e3, "steps": args.steps, "warmup": args.warmup, "dtype": args.dtype,
            "work": "algorithmic (bank prebuilt, no discarded pose pass)" if args.algorithmic else "as executed by the reference",
            "gflop_per_frame_step": gf, "tflops": gf * B / sec / 1e3, "frames": B, "latent": L,
            "finite": bool(torch.isfinite(x).all()), "device": torch.cuda.get_device_name(0) if on_gpu else "cpu"}

    batches = [int(v) for v in str(args.batch).split(",")]
    res = [one(B) for B in batches]
    print(json.dumps(res[0] if len(res) == 1 else {"runs": res}))


if __name__ == "__main__":
    main()
