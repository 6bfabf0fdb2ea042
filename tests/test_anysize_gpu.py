"""Latents whose pixels do not tile into the implicit-GEMM conv's 128-pixel TMA boxes, on the GPU: the 3x3 convs run
on TMA im2col loads (ops.conv3x3_igemm), never on an im2col3x3 buffer.  Portrait 112x64 (a 512x896 image) inference
against the CPU oracle, the drop-in sampler's graph replay against its eager loop, one training step against the
restatement's fp32 autograd at the 64x64 gates of tests/test_train_gpu.py, the training step at 40x24 (no level tiles)
against the unmodified reference's golden at grad16's gates with bit-equal repeats and no im2col kernel in its profile,
and a 4-sample step at 112x64."""
import pytest
import torch

from oracle import restatement as R
from tests import golden_util as G
from tests.test_train_cpu import TRAINED, stage2_model, train_step

pytestmark = pytest.mark.gpu


@pytest.fixture
def no_im2col_buffer(monkeypatch):
    """every 3x3 conv of these sizes must take the im2col-mode TMA loads, not an explicit im2col3x3 + GEMM"""
    from magicdance_b200 import ops

    def refuse(*a, **k):
        raise AssertionError("im2col3x3 launched for a UNet conv")

    monkeypatch.setattr(ops, "im2col3x3", refuse)


def _inputs(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    pose = (torch.rand(b, 3, 8 * h, 8 * w, generator=g) > 0.97).float() * torch.rand(b, 3, 8 * h, 8 * w, generator=g)
    return {"x": torch.randn(b, 4, h, w, generator=g), "ref": 0.8 * torch.randn(b, 4, h, w, generator=g), "pose": pose,
            "context": torch.randn(b, 77, 768, generator=g), "x0": 0.9 * torch.randn(b, 4, h, w, generator=g),
            "noise": torch.randn(b, 4, h, w, generator=g), "t_train": torch.randint(0, 1000, (b,), generator=g)}


def test_portrait_inference_matches_cpu_oracle(no_im2col_buffer):
    from magicdance_b200 import synth
    from magicdance_b200.engine import DenoiseEngine
    sd = synth.synth_state_dict(seed=0)
    inp = _inputs(1, 112, 64, seed=5)
    t = torch.tensor([621])
    with torch.no_grad():
        eng = DenoiseEngine(sd, device="cuda")
        e_gpu = eng.apply_model(inp["x"].cuda(), t.cuda(), inp["context"].cuda(), inp["pose"].cuda(),
                                inp["ref"].cuda(), uc=False)
        del eng
        e_ref = R.apply_model(sd, inp["x"], t, inp["context"], inp["pose"], inp["ref"], uc=False)
    err = G.rel_l2(e_gpu, e_ref)
    print(f"112x64 eps rel-L2 {err:.3e}")
    assert err <= 5e-3


@pytest.fixture(scope="module")
def model():
    m = stage2_model("cuda")
    yield m
    del m
    torch.cuda.empty_cache()


def test_portrait_training_step_against_fp32_autograd(model, no_im2col_buffer):
    """B = 1 at 112x64: loss within 5e-3, d_x_noisy within 1e-2 and every gradient the grad16 golden reaches within
    2e-2 rel-L2 of the restatement's fp32 p_losses autograd (the 64x64 gates)"""
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        inp = _inputs(1, 112, 64, seed=41)
        gold = G.load("grad16")
        reached = [str(n) for n, h, g in zip(gold["names"], gold["has_grad"], gold["gnorm"]) if h and float(g) > 0]
        loss, _, dx, grads = train_step(model, inp)
        sd = {k: v.detach().clone().requires_grad_(k.startswith(TRAINED)) for k, v in model.state_dict().items()
              if v.is_floating_point()}
        dev = {k: v.cuda() for k, v in inp.items()}
        x_noisy = R.q_sample(dev["x0"], dev["t_train"], dev["noise"],
                             R.make_schedule()["alphas_cumprod"]).requires_grad_()
        with torch.enable_grad():
            rl, _, _ = R.p_losses(sd, dev["x0"], dev["t_train"], dev["noise"], dev["context"], dev["pose"],
                                  dev["ref"], x_noisy=x_noisy)
            rl.backward()
        ref = {k: sd[k].grad for k in reached}
        rdx = x_noisy.grad
        del sd
        errs = {k: G.rel_l2(grads[k], ref[k]) for k in reached}
        worst = max(errs, key=errs.get)
        e_dx = G.rel_l2(dx, rdx)
        print(f"112x64: loss {float(loss.detach()):.6f} vs {float(rl.detach()):.6f}; d_x_noisy {e_dx:.3e}; "
              f"worst parameter {worst} {errs[worst]:.3e}")
        assert abs(float(loss) - float(rl)) <= 5e-3 * float(rl)
        assert e_dx <= 1e-2 and errs[worst] <= 2e-2
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
        model.zero_grad(set_to_none=True)
        torch.cuda.empty_cache()


def test_sample_log_graph_replay_matches_eager_at_portrait(model, no_im2col_buffer):
    """the drop-in DDIMSampler_ReferenceOnly.sample (what sample_log runs) with a (4, 112, 64) shape: its graph replay
    (step graph + timestep-batched bank graph) against its eager per-step loop over a 4-step chain at CFG 7"""
    from magicdance_b200.dropin.ddim import DDIMSampler_ReferenceOnly
    inp = {k: v.cuda() for k, v in _inputs(1, 112, 64, seed=11).items()}
    uc_ctx = torch.randn(1, 77, 768, generator=torch.Generator().manual_seed(9)).cuda()
    c = {"c_concat": [inp["pose"]], "c_crossattn": [inp["context"]], "image_control": [inp["ref"]], "wonoise": True,
         "overlap_sampling": False}
    uc = {"c_concat": [inp["pose"]], "c_crossattn": [uc_ctx], "wonoise": True, "overlap_sampling": False}
    model.eval()
    out = []
    try:
        with torch.no_grad():
            for graphs in (True, False):
                sampler = DDIMSampler_ReferenceOnly(model)
                sampler.use_graphs = graphs
                x, _ = sampler.sample(4, 1, (4, 112, 64), c, verbose=False, eta=0.0, x_T=inp["x"],
                                      unconditional_guidance_scale=7.0, unconditional_conditioning=uc)
                out.append(x)
        assert len(model.__dict__.get("_mdb_graphs", {})) == 1  # the graphed path was taken
    finally:
        model.__dict__.pop("_mdb_graphs", None)
        model.__dict__.pop("_mdb_pipelines", None)
        model.train()
        torch.cuda.empty_cache()
    err = G.rel_l2(out[0], out[1])
    print(f"112x64 sampler chain, graphs vs eager: {err:.3e}")
    assert err <= 2e-3


def test_training_at_40x24_matches_the_reference_golden(model, no_im2col_buffer):
    """40x24 (no level tiles into TMA boxes), B = 2: p_losses and the gradients against the UNMODIFIED reference's
    (tests/golden/anysize40x24.npz) at grad16's gates; a repeat is bit-equal; and the profiled step launches no im2col
    kernel of the library (neither ops.im2col3x3 nor one the library would start on its own)"""
    from tests import anysize_golden as A
    from tests.test_train_cpu import TOL
    gold, inp = A.load()
    inp = {k: inp[k] for k in ("x0", "noise", "t_train", "context", "pose", "ref")}
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        a = train_step(model, inp)
        torch.cuda.synchronize()
    kernels = {e.key for e in prof.key_averages()}
    assert any("gemm_igemm_kernel" in k for k in kernels) and any("gemm_bwd_igemm_kernel" in k for k in kernels)
    assert not [k for k in kernels if "im2col3x3" in k], sorted(k for k in kernels if "im2col" in k)
    b = train_step(model, inp)
    A.compare_grads(gold, a[0].detach(), a[2], a[3], TOL)
    assert torch.isfinite(a[0]) and torch.equal(a[0], b[0]) and torch.equal(a[2], b[2])
    for k, g in a[3].items():
        assert (g is None) == (b[3][k] is None) and (g is None or torch.equal(g, b[3][k])), k
    model.zero_grad(set_to_none=True)


def test_four_sample_portrait_step_fits():
    """stage 2, bs 4 at 112x64 (512x896 pose maps), checkpointing, AdamW: one step, finite, peak memory printed"""
    m = stage2_model("cuda")
    opt = torch.optim.AdamW([p for p in m.parameters() if p.requires_grad], lr=1e-5)
    torch.cuda.reset_peak_memory_stats()
    loss, _, dx, grads = train_step(m, _inputs(4, 112, 64, seed=9))
    opt.step()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() / 2**30
    print(f"112x64 bs 4 step: loss {float(loss):.5f}, peak allocated {peak:.1f} GiB")
    assert torch.isfinite(loss) and torch.isfinite(dx).all()
    assert all(torch.isfinite(g).all() for g in grads.values() if g is not None)
    assert peak < 0.9 * torch.cuda.get_device_properties(0).total_memory / 2**30
    del m, opt
    torch.cuda.empty_cache()
