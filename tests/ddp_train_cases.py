"""Data-parallel training as train_tiktok.py:971-976,1002-1009,1212-1239 wires it, run by one process per rank and
checked inside it: DDP(broadcast_buffers=False, bucket_cap_mb=128, find_unused_parameters=True,
gradient_as_bucket_view=True) around the drop-in model, ZeroRedundancyOptimizer(AdamW, weight_decay 0) over the
--finetune_control parameters, `loss, _ = model(x, cond)`, backward, clip_grad_norm_(model.parameters(), 0.5) (the
bf16 path, where the GradScaler is disabled), step, zero_grad(set_to_none=True).

After every step each rank checks:
  a. every parameter, trained or frozen, is bit-equal across ranks (SHA-1 of its bytes, gathered);
  b. the gradient DDP averaged equals the single-process gradient of the concatenated batch, with the same per-sample
     t and noise, taken on this rank from the same weights by torch.autograd.grad (which leaves .grad and DDP's
     hooks alone);
  c. the parameters whose .grad DDP populated are those the single-process gradient reaches (the rest stay None);
  d. sample_log under no_grad gives the same latents as the same call after every library cache was dropped;
  e. no collective is issued from a frame of the magicdance_b200 package, and no library cache holds a CPU tensor
     in shared memory or a tensor on another device.
Checkpointing is on in step 1 and off in step 2, so the reducer sees both graphs.  Ranks build their weights from
different seeds: DDP's construction-time broadcast makes them equal, and d is checked right after it, before any
training forward.  Not a test module: tests/test_train_ddp_gloo.py and tests/test_train_ddp_gpu.py spawn it."""
import hashlib
import os
import socket
import sys
import traceback

import torch
import torch.distributed as dist

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
YAML = {1: os.path.join(REPO, "model_lib", "ControlNet", "models", "cldm_v15_reference_only.yaml"),
        2: os.path.join(REPO, "model_lib", "ControlNet", "models", "cldm_v15_reference_only_pose.yaml")}
NETS = ("unet_config", "control_stage_config", "appearance_control_stage_config", "pose_control_stage_config")
COLLECTIVES = ("all_reduce", "broadcast", "all_gather", "all_gather_into_tensor", "all_gather_object", "reduce",
               "reduce_scatter", "reduce_scatter_tensor", "broadcast_object_list", "gather", "scatter", "barrier",
               "all_to_all", "all_to_all_single", "send", "recv", "isend", "irecv")


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def build_model(stage, seed, small, device):
    """the stage's yaml without the VAE and text encoder (not on this path), synthetic weights from `seed`, and the
    --finetune_control freeze of train_tiktok.py:798-822.  small: 128 model channels at multipliers 1, 2, 2, 2 (the
    inference GroupNorm takes 128 channels or a multiple of 256), 2 heads, a 64-wide context.
    Returns (model, the parameters train_tiktok.py hands to the optimizer)."""
    from magicdance_b200 import synth
    from magicdance_b200.dropin.util import instantiate_from_config, load_config
    cfg = load_config(YAML[stage]).model
    p = cfg["params"]
    p["first_stage_config"], p["cond_stage_config"] = "__is_first_stage__", "__is_unconditional__"
    if small:
        for key in NETS:
            if key in p:
                p[key]["params"].update(model_channels=128, channel_mult=[1, 2, 2, 2], num_heads=2, context_dim=64)
    model = instantiate_from_config(cfg)
    own = model.state_dict()
    sd = synth.synth_state_dict({k: list(v.shape) for k, v in own.items() if k not in synth.SCHEDULE_KEYS}, seed=seed)
    sd.update({k: own[k] for k in synth.SCHEDULE_KEYS})
    model.load_state_dict(sd, strict=True)
    dm = model.model.diffusion_model
    for blk in list(dm.input_blocks) + [dm.middle_block] + list(dm.output_blocks) + list(dm.out):
        blk.requires_grad_(False)
    if stage == 2:
        params = list(model.appearance_control_model.parameters()) + list(model.pose_control_model.parameters())
    else:
        params = list(model.control_model.parameters())
    return model.to(device).train(), params


def batch(n, latent, ctx_dim, seed):
    """n samples: x0, reference latent, pose map, context"""
    g = torch.Generator().manual_seed(seed)
    u, v = torch.rand(n, 3, 8 * latent, 8 * latent, generator=g), torch.rand(n, 3, 8 * latent, 8 * latent, generator=g)
    return {"x0": 0.9 * torch.randn(n, 4, latent, latent, generator=g),
            "ref": 0.8 * torch.randn(n, 4, latent, latent, generator=g),
            "pose": torch.where(u > 0.97, v, torch.zeros_like(v)),
            "context": torch.randn(n, 77, ctx_dim, generator=g)}


def cond_of(inp):
    return {"c_concat": [inp["pose"]], "c_crossattn": [inp["context"]], "image_control": [inp["ref"]], "wonoise": True}


def drop_caches(model):
    """every cache the library keeps on the model and its networks"""
    for key in [k for k in model.__dict__ if k.startswith("_mdb_")]:
        del model.__dict__[key]
    model._engine = None
    for net in model._nets():
        if net is not None:
            net.invalidate()
            net.__dict__.pop("_mdb_train_cache", None)


def sample(model, inp):
    """a 2-step DDIM sample_log at CFG 7 of the first sample, as train_tiktok.py:437-444 calls it"""
    latent = inp["x0"].shape[-1]
    c = dict(cond_of({k: v[:1] for k, v in inp.items()}), overlap_sampling=False)
    uc = {"c_concat": c["c_concat"], "c_crossattn": [torch.zeros_like(inp["context"][:1])], "wonoise": True,
          "overlap_sampling": False}
    x_t = torch.randn(1, 4, latent, latent, generator=torch.Generator().manual_seed(3)).to(inp["x0"].device)
    model.image_size = latent
    with torch.no_grad():
        x, _ = model.sample_log(c, 1, ddim=True, ddim_steps=2, eta=0.0, unconditional_guidance_scale=7.0,
                                unconditional_conditioning=uc, x_T=x_t)
    return x


def check_sample_is_current(model, inp):
    """property d: the cached path against the same call with every cache dropped; returns the latents"""
    x = sample(model, inp)
    drop_caches(model)
    fresh = sample(model, inp)
    assert torch.equal(x, fresh), "sample_log used stale weights"
    return x


def count_library_collectives():
    """wraps torch.distributed's collectives; the returned list collects the ones called from the library"""
    calls = []

    def wrap(name, fn):
        def collective(*a, **k):
            f = sys._getframe(1)
            while f is not None:
                if os.sep + "magicdance_b200" + os.sep in f.f_code.co_filename:
                    calls.append((name, f.f_code.co_filename, f.f_lineno))
                    break
                f = f.f_back
            return fn(*a, **k)
        return collective

    for name in COLLECTIVES:
        setattr(dist, name, wrap(name, getattr(dist, name)))
    return calls


def check_caches_local(model, device):
    """property e: library caches hold tensors of this process, on this rank's device"""
    from magicdance_b200 import ops

    def tensors(o, depth=0):
        if isinstance(o, torch.Tensor):
            yield o
        elif depth < 3 and isinstance(o, dict):
            for v in o.values():
                yield from tensors(v, depth + 1)
        elif depth < 3 and isinstance(o, (list, tuple)):
            for v in o:
                yield from tensors(v, depth + 1)

    found = list(tensors(dict(ops._ws_cache)))
    for net in model._nets():
        if net is not None:
            found += list(tensors(net.__dict__.get("_mdb_train_cache", {})))
    assert found, "no library cache was populated"
    for t in found:
        # (is_shared() is always True for a CUDA tensor: only a CPU tensor can be in shared memory)
        assert (t.is_cuda or not t.is_shared()) and t.device == torch.device(device), (t.shape, t.device)


def param_hashes(model):
    return {k: hashlib.sha1(p.detach().cpu().contiguous().numpy().tobytes()).hexdigest()
            for k, p in model.named_parameters()}


def rel_err(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def train_worker(rank, world, port, backend, stage, small, latent, per_rank, steps, device, q):
    """one rank; puts (rank, None or the failure, report) on q"""
    try:
        q.put((rank, None, _train(rank, world, port, backend, stage, small, latent, per_rank, steps, device)))
    except BaseException:  # the parent reports it
        q.put((rank, traceback.format_exc(), None))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def _train(rank, world, port, backend, stage, small, latent, per_rank, steps, device):
    from torch.distributed.optim import ZeroRedundancyOptimizer
    from torch.nn.parallel import DistributedDataParallel as DDP
    from magicdance_b200 import ops
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group(backend, rank=rank, world_size=world)
    if device == "cpu":
        torch.set_num_threads(max(1, (os.cpu_count() or 1) // world))
        from tests import fake_ops, fake_train_ops
        from tests.test_engine_cpu import _PATCHED
        for name in _PATCHED + ("cfg_ddim_update",):
            setattr(ops, name, getattr(fake_ops, name))
        for name in fake_train_ops.PATCHED:
            setattr(ops, name, getattr(fake_train_ops, name))
    else:
        torch.cuda.set_device(torch.device(device))
    calls = count_library_collectives()
    model, params = build_model(stage, seed=10 + rank, small=small, device=device)
    ctx_dim = 64 if small else 768
    n = world * per_rank
    mine = slice(rank * per_rank, (rank + 1) * per_rank)
    inp = {k: v.to(device) for k, v in batch(n, latent, ctx_dim, seed=7).items()}
    sample(model, inp)  # inference caches packed from this rank's own initial weights
    ddp = DDP(model, device_ids=None if device == "cpu" else [torch.device(device).index], broadcast_buffers=False,
              bucket_cap_mb=128, find_unused_parameters=True, gradient_as_bucket_view=True)
    opt = ZeroRedundancyOptimizer(params, optimizer_class=torch.optim.AdamW, lr=1e-3, weight_decay=0)
    hashes = [None] * world
    dist.all_gather_object(hashes, param_hashes(model))
    assert all(h == hashes[0] for h in hashes), "DDP's construction broadcast left the ranks different"
    x_prev = check_sample_is_current(model, inp)
    trainable = [(k, p) for k, p in model.named_parameters() if p.requires_grad]
    report = {"b_worst_rel_l2": 0.0, "b_worst_param": None, "grads": [], "peak_gib": None}
    seen = {}

    def record(x_start, cond, t, noise=None):  # p_losses as forward() calls it, with its t and noise kept
        noise = torch.randn_like(x_start) if noise is None else noise
        seen["t"], seen["noise"] = t, noise
        return type(model).p_losses(model, x_start, cond, t, noise=noise)

    model.p_losses = record
    for step in range(steps):
        for net in model._nets():
            if net is not None:
                net.use_checkpoint = step == 0
        # parameters that require grad but are not the optimizer's (the UNet's time_embed) keep accumulating .grad
        # across steps: zero_grad clears the optimizer's own only, as in train_tiktok.py
        prior = {k: p.grad.clone() for k, p in trainable if p.grad is not None}
        torch.manual_seed(100 * step + rank)  # t and noise differ per rank, as under torchrun
        loss, _ = ddp(inp["x0"][mine], cond_of({k: v[mine] for k, v in inp.items()}))
        loss.backward()
        # the single-process gradient of the concatenated batch, at the same weights, t and noise
        t_all, noise_all = [torch.empty_like(seen["t"]) for _ in range(world)], [
            torch.empty_like(seen["noise"]) for _ in range(world)]
        dist.all_gather(t_all, seen["t"].contiguous())
        dist.all_gather(noise_all, seen["noise"].contiguous())
        with torch.enable_grad():
            full, _ = type(model).p_losses(model, inp["x0"], cond_of(inp), torch.cat(t_all), noise=torch.cat(noise_all))
            want = torch.autograd.grad(full, [p for _, p in trainable], allow_unused=True)
        reached = {k for (k, _), g in zip(trainable, want) if g is not None}
        populated = {k for k, p in model.named_parameters() if p.grad is not None}
        assert populated == reached, ("c", sorted(populated ^ reached)[:8])
        assert len(reached) < len(trainable)  # the appearance net's layers after its last norm1 stay None
        for (k, p), g in zip(trainable, want):
            if g is not None:
                e = rel_err(p.grad, g + prior[k] if k in prior else g)
                if e > report["b_worst_rel_l2"]:
                    report["b_worst_rel_l2"], report["b_worst_param"] = e, k
        report["grads"].append(len(populated))
        del full, want
        check_caches_local(model, device)
        torch.nn.utils.clip_grad_norm_(ddp.parameters(), 0.5)
        opt.step()
        opt.zero_grad(set_to_none=True)
        dist.all_gather_object(hashes, param_hashes(model))
        assert all(h == hashes[0] for h in hashes), ("a", step)
        x = check_sample_is_current(model, inp)
        assert not torch.equal(x, x_prev), "the step did not change what sample_log computes"
        x_prev = x
    assert not calls, ("e", calls[:4])
    if device != "cpu":
        report["peak_gib"] = torch.cuda.max_memory_allocated() / 2 ** 30
    return report


def run(world, backend, stage, small, latent, per_rank, steps, device, timeout=900):
    """spawns `world` ranks; returns their reports in rank order, raising the first failure"""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=train_worker,
                         args=(r, world, port, backend, stage, small, latent, per_rank, steps, device, q))
             for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = sorted((q.get(timeout=timeout) for _ in range(world)), key=lambda r: r[0])
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
    for rank, err, _ in res:
        assert err is None, f"rank {rank}:\n{err}"
    return [r[2] for r in res]
