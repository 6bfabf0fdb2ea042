"""The training forward and backward on the sm_90a kernels (magicdance_b200/train.py through the drop-in p_losses):
parity with the UNMODIFIED reference's gradients (grad16.npz), precision at the 512x512 training shape against the
restatement's fp32 autograd, determinism (repeat, checkpointing, autocast), inference after an optimizer step, and one
step at BASELINE config 5 (bs 4, latent 64x64)."""
import pytest
import torch

from oracle import restatement as R
from tests import golden_util as G
from tests.test_train_cpu import TRAINED, TOL, compare_to_grad16, stage2_model, train_step

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    m = stage2_model("cuda")
    yield m
    del m
    torch.cuda.empty_cache()


def _inputs(b, latent, seed):
    from magicdance_b200 import synth
    inp = synth.synth_inputs(b, latent, seed=seed, shared_reference=False)
    g = torch.Generator().manual_seed(seed + 1)
    inp["x0"] = 0.9 * torch.randn(b, 4, latent, latent, generator=g)
    inp["noise"] = torch.randn(b, 4, latent, latent, generator=g)
    inp["t_train"] = torch.randint(0, 1000, (b,), generator=g)
    return inp


def test_grad16_parity_with_the_reference(model):
    loss, ld, dx, grads = train_step(model)
    assert set(ld) == {"train/loss_simple", "train/loss_vlb", "train/loss"}
    print("grad16 worst:", compare_to_grad16(loss, dx, grads, TOL))


def test_determinism_checkpointing_and_autocast_are_bit_equal(model):
    runs = [train_step(model), train_step(model), train_step(model, checkpointing=False)]
    with torch.autocast("cuda", dtype=torch.bfloat16):
        runs.append(train_step(model))
    ref = runs[0]
    for r in runs[1:]:
        assert torch.equal(r[0], ref[0]) and torch.equal(r[2], ref[2])
        for k, g in ref[3].items():
            assert (g is None) == (r[3][k] is None) and (g is None or torch.equal(g, r[3][k])), k


def test_precision_at_64x64_against_fp32_autograd(model):
    """latent 64x64 (512x512 image), no scaler: every gradient the golden reaches within 2e-2 rel-L2 of the
    restatement's fp32 p_losses autograd on the same GPU, d_x_noisy within 1e-2; then the GradScaler leg.  B = 1: the
    restatement's fp32 autograd keeps every attention map, and two samples of it do not fit beside the model."""
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False  # an fp32 reference
    try:
        _precision_64(model)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32


def _precision_64(model):
    inp = _inputs(1, 64, seed=41)
    gold = G.load("grad16")
    reached = [str(n) for n, h, g in zip(gold["names"], gold["has_grad"], gold["gnorm"]) if h and float(g) > 0]
    loss, _, dx, grads = train_step(model, inp)
    sd = {k: v.detach().clone().requires_grad_(k.startswith(TRAINED)) for k, v in model.state_dict().items()
          if v.is_floating_point()}  # the model's own weights
    dev = {k: v.cuda() for k, v in inp.items()}
    x_noisy = R.q_sample(dev["x0"], dev["t_train"], dev["noise"], R.make_schedule()["alphas_cumprod"]).requires_grad_()
    with torch.enable_grad():
        rl, _, _ = R.p_losses(sd, dev["x0"], dev["t_train"], dev["noise"], dev["context"], dev["pose"], dev["ref"],
                              x_noisy=x_noisy)
        rl.backward()
    ref = {k: sd[k].grad for k in reached}
    rdx = x_noisy.grad
    del sd
    errs = {k: G.rel_l2(grads[k], ref[k]) for k in reached}
    worst = max(errs, key=errs.get)
    e_dx = G.rel_l2(dx, rdx)
    print(f"64x64: loss {float(loss):.6f} vs {float(rl):.6f}; d_x_noisy {e_dx:.3e}; worst parameter {worst} "
          f"{errs[worst]:.3e}")
    assert abs(float(loss) - float(rl)) <= 5e-3 * float(rl)
    assert e_dx <= 1e-2 and errs[worst] <= 2e-2
    # GradScaler: scaler.scale(loss).backward() gives S times the gradients
    S = 65536.0
    _, _, sdx, sgrads = train_step(model, inp, scale=S)
    serrs = {k: G.rel_l2(sgrads[k] / S, ref[k]) for k in reached}
    sw = max(serrs, key=serrs.get)
    print(f"64x64 with a x{S:g} loss scale: d_x_noisy {G.rel_l2(sdx / S, rdx):.3e}; worst parameter {sw} "
          f"{serrs[sw]:.3e}")
    assert G.rel_l2(sdx / S, rdx) <= 1e-2 and serrs[sw] <= 2e-2


def _fresh_copy(model):
    m = stage2_model("cpu")
    m.load_state_dict(model.state_dict())
    return m.to("cuda")


def _eps(m, inp):
    dev = {k: v.cuda() for k, v in inp.items()}
    cond = {"c_concat": [dev["pose"]], "c_crossattn": [dev["context"]]}
    with torch.no_grad():
        return m.apply_model(dev["x"], dev["t_train"], cond, dev["ref"])


def test_inference_after_training_sees_the_new_weights(model):
    inp = _inputs(2, 32, seed=7)  # the inference engine needs 8-token multiples at the deepest level
    before = _eps(model, inp)
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-3)
    train_step(model)
    opt.step()
    after = _eps(model, inp)
    assert not torch.equal(after, before)
    fresh = _fresh_copy(model)
    assert torch.equal(after, _eps(fresh, inp))
    del fresh
    # an update the version counters do not see, then a training call
    with torch.no_grad():
        for p in model.pose_control_model.parameters():
            p.data.copy_(p.data * 0.5)
    train_step(model)
    fresh = _fresh_copy(model)
    assert torch.equal(_eps(model, inp), _eps(fresh, inp))
    del fresh, opt
    model.load_state_dict(stage2_model("cpu").state_dict())  # the weights the other tests expect
    model.zero_grad(set_to_none=True)


def test_config5_step_runs_with_finite_gradients():
    """BASELINE config 5: bs 4, 64x64 latent, 512x512 pose maps, AdamW; one step, peak memory printed"""
    m = stage2_model("cuda")
    opt = torch.optim.AdamW([p for p in m.parameters() if p.requires_grad], lr=1e-5)
    torch.cuda.reset_peak_memory_stats()
    loss, _, dx, grads = train_step(m, _inputs(4, 64, seed=3))
    opt.step()
    torch.cuda.synchronize()
    print(f"config 5 step: loss {float(loss):.5f}, peak allocated {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
    assert torch.isfinite(loss) and torch.isfinite(dx).all()
    assert all(torch.isfinite(g).all() for g in grads.values() if g is not None)
    assert all(torch.isfinite(p).all() for p in m.parameters() if p.requires_grad)
    del m, opt
    torch.cuda.empty_cache()
