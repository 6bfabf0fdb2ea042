"""The training forward's orchestration on the CPU (magicdance_b200/train.py through the drop-in p_losses): the autograd
ops are replaced by the layout-checking, fp16-rounding PyTorch stand-ins of tests/fake_train_ops.py, and loss.backward()
at the grad16 inputs is held to the gradients the UNMODIFIED reference produced (tests/golden/grad16.npz: stage-2
freeze, CheckpointFunction active)."""
import os

import numpy as np
import pytest
import torch

from tests import golden_util as G

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
YAML = os.path.join(REPO, "model_lib", "ControlNet", "models", "cldm_v15_reference_only_pose.yaml")
TRAINED = ("appearance_control_model.", "pose_control_model.")


def stage2_model(device="cpu"):
    """create_model(yaml) with the synthetic weights of the goldens and the freeze of train_tiktok.py:798-822
    (--finetune_control): the SD UNet's input / middle / output blocks and `out` frozen"""
    from magicdance_b200 import synth
    from model_lib.ControlNet.cldm.model import create_model
    model = create_model(YAML)
    sd = synth.synth_state_dict(seed=0)
    own = model.state_dict()
    sd.update({k: own[k] for k in synth.SCHEDULE_KEYS})
    sd.update({k: own[k] for k in own if k.startswith("first_stage_model.")})
    missing, unexpected = model.load_state_dict(sd, strict=True)
    assert not missing and not unexpected
    dm = model.model.diffusion_model
    for blk in list(dm.input_blocks) + [dm.middle_block] + list(dm.output_blocks) + list(dm.out):
        for p in blk.parameters():
            p.requires_grad_(False)
    return model.to(device).train()


def train_step(model, inp=None, checkpointing=True, scale=1.0):
    """p_losses + backward (of scale * loss) at `inp` (default: the grad16 inputs), x_noisy's gradient taken as
    oracle/make_golden_grad.py takes it.  Returns (loss, loss_dict, d_x_noisy, {trained name: grad or None})."""
    dev = model.device
    inp = {k: v.to(dev) for k, v in (inp or G.grad16_inputs()).items()}
    for net in (model.model.diffusion_model, model.appearance_control_model, model.pose_control_model):
        net.use_checkpoint = checkpointing
    model.zero_grad(set_to_none=True)
    probe = {}
    fwd = model.apply_model

    def rec(x_noisy, *a, **k):
        x_noisy.requires_grad_(True)
        probe["x"] = x_noisy
        return fwd(x_noisy, *a, **k)

    cond = {"c_concat": [inp["pose"]], "c_crossattn": [inp["context"]], "image_control": [inp["ref"]], "wonoise": True}
    model.apply_model = rec
    try:
        with torch.enable_grad():
            loss, ld = model.p_losses(inp["x0"], cond, inp["t_train"], noise=inp["noise"])
            (loss * scale).backward()
    finally:
        del model.apply_model
    grads = {k: (None if p.grad is None else p.grad.detach().clone()) for k, p in model.named_parameters()
             if k.startswith(TRAINED)}
    return loss.detach(), ld, probe["x"].grad.detach().clone(), grads


def compare_to_grad16(loss, dx, grads, tol):
    """worst errors against grad16.npz, each checked against tol[name]; returns them"""
    gold = G.load("grad16")
    names = [str(n) for n in gold["names"]]
    assert sorted(names) == sorted(grads)
    worst = {"loss": abs(float(loss) - float(gold["loss"])) / float(gold["loss"]),
             "d_x_noisy": G.rel_l2(dx, torch.from_numpy(gold["d_x_noisy"])), "norm": 0.0, "sample": 0.0, "sum": 0.0,
             "full": 0.0}
    reached = {n for n in names if grads[n] is not None and float(grads[n].abs().max()) > 0}
    assert reached == {n for n, h, g in zip(names, gold["has_grad"], gold["gnorm"]) if h and float(g) > 0}
    for i, n in enumerate(names):
        if n not in reached:
            continue
        g = grads[n].double().cpu().flatten()
        norm = float(gold["gnorm"][i])
        worst["norm"] = max(worst["norm"], abs(float(g.norm()) - norm) / norm)
        pos = G.grad_sample_positions(g.numel())
        err = float((g[torch.from_numpy(pos)] - torch.from_numpy(gold["gsample"][i, :len(pos)])).norm()) / (
            norm / np.sqrt(g.numel()) * np.sqrt(len(pos)))
        worst["sample"] = max(worst["sample"], err)
        worst["sum"] = max(worst["sum"], abs(float(g.sum()) - float(gold["gsum"][i])) / (norm * np.sqrt(g.numel())))
    for key in gold.files:
        if key.startswith("full/"):
            worst["full"] = max(worst["full"], G.rel_l2(grads[key[5:]], torch.from_numpy(gold[key])))
    print({k: f"{v:.3e}" for k, v in worst.items()})
    for k, v in worst.items():
        assert v <= tol[k], (k, v, tol[k])
    return worst


TOL = {"loss": 5e-3, "d_x_noisy": 1e-2, "norm": 2e-2, "sample": 3e-2, "sum": 2e-2, "full": 2e-2}


@pytest.fixture(scope="module")
def runs():
    from magicdance_b200 import ops
    from tests import fake_train_ops
    with pytest.MonkeyPatch.context() as mp:
        for name in fake_train_ops.PATCHED:
            mp.setattr(ops, name, getattr(fake_train_ops, name))
        model = stage2_model()
        on = train_step(model, checkpointing=True)
        off = train_step(model, checkpointing=False)
        yield model, on, off


def test_training_forward_and_backward_match_the_reference_gradients(runs):
    _, (loss, ld, dx, grads), _ = runs
    assert set(ld) == {"train/loss_simple", "train/loss_vlb", "train/loss"}
    compare_to_grad16(loss, dx, grads, TOL)


def test_checkpointing_changes_memory_not_values(runs):
    _, on, off = runs
    assert torch.equal(on[0], off[0]) and torch.equal(on[2], off[2])
    for k, g in on[3].items():
        assert (g is None) == (off[3][k] is None), k
        assert g is None or torch.equal(g, off[3][k]), k


def test_frozen_and_unreached_parameters_keep_no_gradient(runs):
    model, (_, _, _, grads), _ = runs
    gold = G.load("grad16")
    dead = {str(n) for n, h in zip(gold["names"], gold["has_grad"]) if not h}
    assert len(dead) == 36 and all(grads[n] is None for n in dead)
    dm = model.model.diffusion_model
    frozen = [p for blk in list(dm.input_blocks) + [dm.middle_block] + list(dm.output_blocks) + list(dm.out)
              for p in blk.parameters()]
    assert frozen and all(p.grad is None for p in frozen)
    assert dm.time_embed[0].weight.grad is not None  # trained in stage 2 (only the blocks are frozen)


def test_frozen_copies_follow_in_place_updates():
    """copies of frozen parameters are cached, keyed on storage and version: an in-place update makes a new copy,
    an unchanged parameter keeps its copy"""
    from magicdance_b200.train import GradScale, _Weights
    m = torch.nn.Conv2d(64, 64, 3)
    m.requires_grad_(False)
    w = _Weights(m, GradScale())
    a16, _ = w.conv("weight")
    assert w.conv("weight")[0] is a16
    with torch.no_grad():
        m.weight.add_(1.0)
    b16, _ = _Weights(m, GradScale()).conv("weight")
    assert b16 is not a16 and torch.equal(b16, (m.weight.permute(0, 2, 3, 1).reshape(64, -1)).half())
    m.weight.requires_grad_(True)  # trained: a fresh copy per forward, through the gradient unscale
    with torch.enable_grad():  # (other modules disable grad globally)
        c16, cp = _Weights(m, GradScale()).conv("weight")
    assert torch.equal(c16, b16) and cp.requires_grad and cp.grad_fn is not None


def test_inference_packing_follows_parameter_updates(monkeypatch):
    """UNetModel.packed(): the same object while the weights are unchanged, a new one after an in-place update (an
    optimizer step bumps the version counters) or invalidate() (an update that bypasses them)"""
    from magicdance_b200 import ops
    from magicdance_b200.dropin.cldm import ControlNet
    from tests import fake_ops
    monkeypatch.setattr(ops, "require_cuda", fake_ops.require_cuda)
    net = ControlNet(image_size=32, in_channels=4, hint_channels=3, model_channels=64, attention_resolutions=[4],
                     num_res_blocks=1, channel_mult=[1, 2], num_heads=2, use_spatial_transformer=True,
                     transformer_depth=1, context_dim=64, legacy=False)
    p1 = net.packed("cpu")
    assert net.packed("cpu") is p1
    with torch.no_grad():
        net.input_blocks[0][0].weight.add_(1.0)
    p2 = net.packed("cpu")
    assert p2 is not p1 and net.packed("cpu") is p2
    with torch.no_grad():
        net.input_blocks[0][0].weight.data.copy_(torch.zeros_like(net.input_blocks[0][0].weight))
    assert net.packed("cpu") is p2  # .data bypasses the version counter ...
    net.invalidate()
    assert net.packed("cpu") is not p2  # ... which is why the training path invalidates the nets it trains


def test_unsupported_latent_sizes_are_refused():
    from magicdance_b200.engine import NetConfig
    from magicdance_b200.train import check_latent_size
    for s in (16, 32, 64):
        check_latent_size(NetConfig(), s, s)
    with pytest.raises(ValueError, match="training forward"):
        check_latent_size(NetConfig(), 12, 12)
