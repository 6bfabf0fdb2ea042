#!/usr/bin/env python
"""BASELINE configs[4] and 5 under torchrun: training throughput of the drop-in model on the library's kernels with
one process per GPU, wrapped as train_tiktok.py:971-976,1002-1009 wraps it.

scripts/train_bench.py's recipe (4 samples per GPU at a 64x64 latent, stage 2 with the --finetune_control freeze, AdamW
at lr 1e-5 over the parameters that require grad, activation checkpointing) inside
DDP(device_ids=[local_rank], broadcast_buffers=False, bucket_cap_mb=128, find_unused_parameters=True,
gradient_as_bucket_view=True) and ZeroRedundancyOptimizer(optimizer_class=AdamW, weight_decay=0); each step is
`loss, _ = model(x, cond)` (t and noise drawn inside, different per rank), backward, clip_grad_norm_(0.5) (the bf16
path, where the GradScaler is disabled), step, zero_grad(set_to_none=True).  Each rank trains on its own samples.

Rank 0 first times train_bench.py's plain single-process loop in the same run (no DDP, no ZeRO, no clip), so the
overhead of the wrapping is a measured number.  Prints one JSON line from rank 0: world size, the card and its power
limit (read in the same run from `nvidia-smi --query-gpu`), total and per-GPU samples/s, ms/step, peak allocated memory
of every rank, and the plain loop's numbers.  --profile DIR adds a separate torch.profiler pass over the DDP loop
(traces written under DIR) and reports its NCCL kernel time and the part of it no compute kernel overlaps.  Writes
nothing to the tree.

    torchrun --nproc-per-node 8 scripts/train_ddp_bench.py [--stage 2] [--batch 4] [--steps 5] [--warmup 2]
                                                          [--profile DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "scripts"))


def _wrap(model, local_rank):
    import torch
    from torch.distributed.optim import ZeroRedundancyOptimizer
    from torch.nn.parallel import DistributedDataParallel as DDP
    ddp = DDP(model, device_ids=[local_rank], output_device=local_rank, broadcast_buffers=False, bucket_cap_mb=128,
              find_unused_parameters=True, gradient_as_bucket_view=True)
    opt = ZeroRedundancyOptimizer([p for p in model.parameters() if p.requires_grad],
                                  optimizer_class=torch.optim.AdamW, lr=1e-5, weight_decay=0)
    return ddp, opt


def _inputs(batch, latent, rank):
    import torch
    from magicdance_b200 import synth
    inp = {k: v.cuda() for k, v in synth.synth_inputs(batch, latent, seed=rank, shared_reference=False).items()}
    g = torch.Generator(device="cuda").manual_seed(rank)
    cond = {"c_concat": [inp["pose"]], "c_crossattn": [inp["context"]], "image_control": [inp["ref"]], "wonoise": True}
    return 0.9 * torch.randn(batch, 4, latent, latent, device="cuda", generator=g), cond


def _step(ddp, opt, x0, cond):
    import torch
    loss, _ = ddp(x0, cond)
    loss.backward()
    torch.nn.utils.clip_grad_norm_(ddp.parameters(), 0.5)
    opt.step()
    opt.zero_grad(set_to_none=True)
    return loss


def run_ddp(ddp, opt, x0, cond, steps, warmup):
    import torch
    import torch.distributed as dist
    for _ in range(warmup):
        _step(ddp, opt, x0, cond)
    torch.cuda.synchronize()
    dist.barrier()
    torch.cuda.reset_peak_memory_stats()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        loss = _step(ddp, opt, x0, cond)
    end.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(end) / steps
    return ms, torch.cuda.max_memory_allocated() / 2 ** 30, bool(torch.isfinite(loss))


def _intervals_total(iv):
    total, cur_s, cur_e = 0.0, None, None
    for s, e in sorted(iv):
        if cur_e is None or s > cur_e:
            if cur_e is not None:
                total += cur_e - cur_s
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    return total + (0.0 if cur_e is None else cur_e - cur_s)


def profile_nccl(ddp, opt, x0, cond, steps, out_dir, rank):
    """NCCL kernel time per step, and the part of it during which no other kernel runs (from kernel intervals)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    os.makedirs(out_dir, exist_ok=True)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            _step(ddp, opt, x0, cond)
        torch.cuda.synchronize()
    prof.export_chrome_trace(os.path.join(out_dir, f"train_ddp_rank{rank}.pt.trace.json"))
    nccl, compute = [], []
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA or ev.time_range.elapsed_us() <= 0:
            continue
        iv = (ev.time_range.start, ev.time_range.end)
        (nccl if "nccl" in ev.name.lower() else compute).append(iv)
    total = _intervals_total(nccl)
    # NCCL time covered by compute = |nccl| + |compute| - |nccl U compute|
    covered = total + _intervals_total(compute) - _intervals_total(nccl + compute)
    return {"nccl_kernel_ms_per_step": total / 1e3 / steps,
            "nccl_not_overlapped_ms_per_step": (total - covered) / 1e3 / steps, "nccl_kernels": len(nccl)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stage", type=int, default=2, choices=(1, 2),
                    help="2: appearance-disentangled pose control; 1: appearance-control pre-training")
    ap.add_argument("--batch", type=int, default=4, help="samples per GPU")
    ap.add_argument("--latent", type=int, default=64)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", default=None, help="directory for a separate torch.profiler pass")
    args = ap.parse_args()
    import torch
    import torch.distributed as dist
    import train_bench
    assert torch.cuda.is_available(), "needs an sm_90 GPU"
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    rank, world = dist.get_rank(), dist.get_world_size()
    model = train_bench.build_model(args.stage)
    for net in (n for n in model._nets() if n is not None):
        net.use_checkpoint = True
    out = {}
    if rank == 0:
        name, limit = train_bench.gpu_info()
        out = {"metric": f"training samples/s under DDP + ZeRO (stage {args.stage}, torchrun)", "world_size": world,
               "device": name, "power_limit_w": limit, "batch_per_gpu": args.batch, "latent": args.latent,
               "steps": args.steps, "warmup": args.warmup}
        # the plain loop before DDP's broadcast: rank 0's weights are the ones every rank trains from
        out["plain_world1"] = train_bench.run(model, args.batch, args.latent, args.steps, args.warmup,
                                              checkpointing=True)
    dist.barrier()
    x0, cond = _inputs(args.batch, args.latent, rank)
    ddp, opt = _wrap(model, local_rank)
    ms, peak, finite = run_ddp(ddp, opt, x0, cond, args.steps, args.warmup)
    peaks = [None] * world
    dist.all_gather_object(peaks, peak)
    prof = profile_nccl(ddp, opt, x0, cond, args.steps, args.profile, rank) if args.profile else None
    if rank == 0:
        out.update({"samples_per_s": world * args.batch * 1e3 / ms, "samples_per_s_per_gpu": args.batch * 1e3 / ms,
                    "ms_per_step": ms, "peak_allocated_gib_per_rank": peaks, "finite": finite})
        plain = out["plain_world1"]
        if isinstance(plain, dict):
            out["ddp_zero_overhead_ms_per_step"] = ms - plain["ms_per_step"]
        if prof is not None:
            out["profile"] = prof
        print(json.dumps(out))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
