"""train_tiktok.py's data-parallel step (DDP + ZeroRedundancyOptimizer) on one H100 with the library's kernels.

World size 1 over NCCL: after two steps the parameters are bit-equal to the plain single-process loop's.  World size 2
over gloo with both ranks on the one GPU (NCCL takes one rank per device): stage 1 at a 16x16 latent, one sample per
rank, every property tests/ddp_train_cases.py lists, the gradient held against the single-process gradient of the
2-sample batch."""
import os

import pytest
import torch

from tests import ddp_train_cases as D

pytestmark = pytest.mark.gpu

# the per-rank GEMM plans differ from the 2-sample batch's (split-K is chosen from the row count), so the fp16
# activations round differently, beside the fp32 sums in another order
GRAD_REL_L2 = 1e-2


def _need_free_gib(gib):
    free, _ = torch.cuda.mem_get_info()
    if free < gib * 2 ** 30:
        pytest.skip(f"{free / 2 ** 30:.1f} GiB free on the GPU, {gib} GiB needed")


def _step(ddp_or_model, model, opt, inp):
    loss, _ = ddp_or_model(inp["x0"], D.cond_of(inp))
    loss.backward()
    torch.nn.utils.clip_grad_norm_(ddp_or_model.parameters(), 0.5)
    opt.step()
    opt.zero_grad(set_to_none=True)


def _ddp_world1(q):
    from torch.distributed.optim import ZeroRedundancyOptimizer
    from torch.nn.parallel import DistributedDataParallel as DDP
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(D.free_port())
    try:
        dist.init_process_group("nccl", rank=0, world_size=1)
        torch.cuda.set_device(0)
        model, params = D.build_model(2, seed=0, small=False, device="cuda")
        init = {k: v.clone() for k, v in model.state_dict().items()}
        inp = {k: v.cuda() for k, v in D.batch(2, 16, 768, seed=7).items()}
        plain = torch.optim.AdamW(params, lr=1e-5, weight_decay=0)
        for step in range(2):
            torch.manual_seed(step)
            _step(model, model, plain, inp)
        want = {k: p.detach().clone() for k, p in model.named_parameters()}
        del plain
        model.zero_grad(set_to_none=True)
        model.load_state_dict(init)
        ddp = DDP(model, device_ids=[0], broadcast_buffers=False, bucket_cap_mb=128, find_unused_parameters=True,
                  gradient_as_bucket_view=True)
        opt = ZeroRedundancyOptimizer(params, optimizer_class=torch.optim.AdamW, lr=1e-5, weight_decay=0)
        for step in range(2):
            torch.manual_seed(step)
            _step(ddp, model, opt, inp)
        differ = [k for k, p in model.named_parameters() if not torch.equal(p, want[k])]
        moved = sum(not torch.equal(want[k], init[k]) for k in want)
        q.put((differ, moved, torch.cuda.max_memory_allocated() / 2 ** 30))
    except BaseException:
        import traceback
        q.put(traceback.format_exc())
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def test_ddp_zero_world1_nccl_equals_the_plain_loop():
    _need_free_gib(50)
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    p = ctx.Process(target=_ddp_world1, args=(q,))
    p.start()
    try:
        res = q.get(timeout=900)
    finally:
        p.join(timeout=60)
        if p.is_alive():
            p.kill()
    assert not isinstance(res, str), res
    differ, moved, peak = res
    print(f"world 1 NCCL, stage 2, 2 samples at 16x16: peak allocated {peak:.1f} GiB; {moved} parameters moved")
    assert moved > 0 and differ == []


def test_ddp_zero_world2_gloo_one_gpu_stage1():
    _need_free_gib(50)
    reports = D.run(2, "gloo", 1, small=False, latent=16, per_rank=1, steps=2, device="cuda:0")
    worst = max(r["b_worst_rel_l2"] for r in reports)
    name = max(reports, key=lambda r: r["b_worst_rel_l2"])["b_worst_param"]
    for rank, r in enumerate(reports):
        print(f"rank {rank}: peak allocated {r['peak_gib']:.1f} GiB; gradients populated per step {r['grads']}")
    print(f"worst per-parameter gradient rel-L2 against the 2-sample single-process gradient {worst:.3e} ({name})")
    assert worst <= GRAD_REL_L2
    assert reports[0]["grads"] == reports[1]["grads"]
