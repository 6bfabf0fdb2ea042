#!/usr/bin/env python
"""BASELINE config 5 on one GPU: training throughput of the drop-in model on the library's kernels.

SURVEY §8 recipe: a synthetic batch of 4 samples at a 64x64 latent (512x512 pose maps), t ~ U{0..999} per sample, AdamW
at lr 1e-5, the appearance net and the pose ControlNet trained, the SD UNet frozen (train_tiktok.py:798-822
--finetune_control: its input / middle / output blocks and `out`); warm-up steps, then timed steps of p_losses ->
backward -> optimizer step between CUDA events.  Runs with activation checkpointing (the yaml's use_checkpoint) and
without it (when it fits in memory).

Prints one JSON line: the card and its power limit (read in the same run from `nvidia-smi --query-gpu`), samples/s,
ms/step and peak allocated memory per mode, and algorithmic TFLOP/s against the 6738.5 GF per sample that
oracle/count_training_flops.py counted on the reference (stage-2 freeze, with the checkpoint recompute).  Writes nothing
to the tree.

With --stage 1 it measures stage-1 appearance-control pre-training instead (models/cldm_v15_reference_only.yaml,
scripts/appearance_control_pretraining.sh: ControlLDMReferenceOnly, the appearance net trained, the same UNet freeze, its
time_embed reached by the gradient); no reference FLOP count is taken for it.

With --latent-hw HxW (e.g. 112x64: a 512x896 portrait frame) it trains at a latent whose sides need not be equal or
tile into the implicit-GEMM conv's TMA boxes (those levels' 3x3 convs run on TMA im2col loads); the reference FLOP
count is for 64x64 and is then not used.

    python scripts/train_bench.py [--stage 2] [--batch 4] [--latent 64 | --latent-hw 112x64] [--steps 5] [--warmup 2]
                                  [--modes ckpt,plain]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

REFERENCE_GF_PER_SAMPLE = 6738.5  # oracle/count_training_flops.py: use_checkpoint True, forward + backward


def gpu_info():
    """(name, power limit in W) of the current card, read-only"""
    import torch
    name, limit = torch.cuda.get_device_name(0), None
    try:
        idx = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0] or "0"
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", idx],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        if out:
            name, limit = [v.strip() for v in out[0].split(",")][:2]
            limit = float(limit)
    except (OSError, subprocess.SubprocessError, ValueError):
        pass
    return name, limit


def build_model(stage=2):
    import torch
    from magicdance_b200 import synth
    from model_lib.ControlNet.cldm.model import create_model
    yaml = "cldm_v15_reference_only_pose.yaml" if stage == 2 else "cldm_v15_reference_only.yaml"
    model = create_model(os.path.join(REPO, "model_lib", "ControlNet", "models", yaml))
    own = model.state_dict()
    if stage == 2:
        sd = synth.synth_state_dict(seed=0)
    else:  # the stage-1 layout: synthesised per key of the model's own state dict
        sd = synth.synth_state_dict({k: list(v.shape) for k, v in own.items()
                                     if k not in synth.SCHEDULE_KEYS and not k.startswith("first_stage_model.")}, seed=0)
    sd.update({k: own[k] for k in own if k not in sd})
    model.load_state_dict(sd, strict=True)
    dm = model.model.diffusion_model
    for blk in list(dm.input_blocks) + [dm.middle_block] + list(dm.output_blocks) + list(dm.out):
        blk.requires_grad_(False)
    return model.to("cuda").train()


def _inputs_hw(batch, h, w):
    """synth_inputs' recipe at an h x w latent"""
    import torch
    g = torch.Generator().manual_seed(0)
    u, v = torch.rand(batch, 3, 8 * h, 8 * w, generator=g), torch.rand(batch, 3, 8 * h, 8 * w, generator=g)
    return {"ref": 0.8 * torch.randn(batch, 4, h, w, generator=g), "pose": torch.where(u > 0.97, v, torch.zeros_like(v)),
            "context": torch.randn(1, 77, 768, generator=g).expand(batch, -1, -1).contiguous()}


def run(model, batch, latent, steps, warmup, checkpointing, latent_hw=None):
    import torch
    from magicdance_b200 import synth
    for net in (n for n in model._nets() if n is not None):
        net.use_checkpoint = checkpointing
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-5)
    if latent_hw is None:
        inp = synth.synth_inputs(batch, latent, seed=0, shared_reference=False)
        h = w = latent
    else:
        h, w = latent_hw
        inp = _inputs_hw(batch, h, w)
    inp = {k: v.cuda() for k, v in inp.items()}
    g = torch.Generator(device="cuda").manual_seed(0)
    cond = {"c_concat": [inp["pose"]], "c_crossattn": [inp["context"]], "image_control": [inp["ref"]], "wonoise": True}
    x0 = 0.9 * torch.randn(batch, 4, h, w, device="cuda", generator=g)

    def step():
        t = torch.randint(0, 1000, (batch,), device="cuda", generator=g)
        loss, _ = model.p_losses(x0, cond, t, noise=torch.randn(x0.shape, device="cuda", generator=g))
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        return loss

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        loss = step()
    end.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(end) / steps
    res = {"samples_per_s": batch * 1e3 / ms, "ms_per_step": ms,
           "peak_allocated_gib": torch.cuda.max_memory_allocated() / 2 ** 30,
           "algorithmic_tflops_vs_reference_count": REFERENCE_GF_PER_SAMPLE * batch / ms,
           "finite": bool(torch.isfinite(loss))}
    if model._nets()[2] is None or latent_hw is not None:  # the reference FLOP count is stage 2's, at 64x64
        del res["algorithmic_tflops_vs_reference_count"]
    del opt
    model.zero_grad(set_to_none=True)
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stage", type=int, default=2, choices=(1, 2),
                    help="2: appearance-disentangled pose control; 1: appearance-control pre-training")
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--latent", type=int, default=64)
    ap.add_argument("--latent-hw", default=None, help="HxW: a latent of H rows and W columns instead of --latent")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--modes", default="ckpt,plain", help="ckpt (activation checkpointing), plain (none)")
    args = ap.parse_args()
    latent_hw = tuple(int(v) for v in args.latent_hw.lower().split("x")) if args.latent_hw else None
    import torch
    assert torch.cuda.is_available(), "needs an sm_90 GPU"
    name, limit = gpu_info()
    model = build_model(args.stage)
    if args.stage == 2:
        out = {"metric": "training samples/s (BASELINE config 5, stage 2, one GPU)", "device": name,
               "power_limit_w": limit, "batch": args.batch, "latent": args.latent, "steps": args.steps,
               "warmup": args.warmup, "reference_gf_per_sample": REFERENCE_GF_PER_SAMPLE}
    else:
        out = {"metric": "training samples/s (stage 1 appearance-control pre-training, one GPU)", "device": name,
               "power_limit_w": limit, "batch": args.batch, "latent": args.latent, "steps": args.steps,
               "warmup": args.warmup}
    if latent_hw is not None:
        out["latent"] = list(latent_hw)
        out.pop("reference_gf_per_sample", None)
    for mode in args.modes.split(","):
        try:
            out[mode] = run(model, args.batch, args.latent, args.steps, args.warmup, checkpointing=mode == "ckpt",
                            latent_hw=latent_hw)
        except torch.cuda.OutOfMemoryError:
            model.zero_grad(set_to_none=True)
            torch.cuda.empty_cache()
            out[mode] = "does not fit in memory"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
