"""Stage-1 appearance-control pre-training (ControlLDMReferenceOnly, models/cldm_v15_reference_only.yaml) through the
drop-in on the CPU: the yaml, the state-dict layout, and — with the kernels replaced by the layout-checking PyTorch
stand-ins of tests/fake_ops.py and tests/fake_train_ops.py — apply_model, the bank, p_losses, a 4-step sample_log chain
against the UNMODIFIED reference's stage-1 model (oracle/make_golden_stage1.py).  The training gradients are checked in
tests/test_stage1_train_cpu.py with the helpers defined here."""
import json
import os

import numpy as np
import pytest
import torch

from tests import golden_util as G

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
YAML = os.path.join(REPO, "model_lib", "ControlNet", "models", "cldm_v15_reference_only.yaml")
YAML_POSE = os.path.join(REPO, "model_lib", "ControlNet", "models", "cldm_v15_reference_only_pose.yaml")
TRAINED = ("control_model.", "model.diffusion_model.time_embed.")
TOL = {"loss": 5e-3, "d_x_noisy": 1e-2, "norm": 2e-2, "sample": 3e-2, "sum": 2e-2, "full": 2e-2}  # as for grad16


def reference_manifest():
    with open(os.path.join(G.GOLDEN, "stage1_manifest.json")) as f:
        return json.load(f)


def synth_weights(model, seed=0):
    """the goldens' synthetic weights for every network key of the model's own layout; schedule buffers and the VAE
    are the model's own"""
    from magicdance_b200 import synth
    own = model.state_dict()
    nets = {k: list(v.shape) for k, v in own.items()
            if k not in synth.SCHEDULE_KEYS and not k.startswith("first_stage_model.")}
    sd = synth.synth_state_dict(nets, seed=seed)
    sd.update({k: v for k, v in own.items() if k in synth.SCHEDULE_KEYS or k.startswith("first_stage_model.")})
    return sd


def freeze_stage1(model):
    """train_tiktok.py:798-801 (--finetune_control): the UNet's input / middle / output blocks and `out` frozen;
    its time_embed stays trainable"""
    dm = model.model.diffusion_model
    for blk in list(dm.input_blocks) + [dm.middle_block] + list(dm.output_blocks) + list(dm.out):
        for p in blk.parameters():
            p.requires_grad_(False)
    return model


def stage1_model(device="cpu", freeze=True):
    from model_lib.ControlNet.cldm.model import create_model
    model = create_model(YAML)
    missing, unexpected = model.load_state_dict(synth_weights(model), strict=True)
    assert not missing and not unexpected
    if freeze:
        freeze_stage1(model)
    return model.to(device)


def train_step(model, inp=None, checkpointing=True, scale=1.0):
    """p_losses + backward of scale * loss, x_noisy's gradient taken as the oracle takes it.  Returns (loss, loss_dict,
    d_x_noisy, {recorded name: grad or None})."""
    dev = model.device
    inp = {k: v.to(dev) for k, v in (inp or G.grad16_inputs()).items()}
    for net in (model.model.diffusion_model, model.control_model):
        net.use_checkpoint = checkpointing
    model.zero_grad(set_to_none=True)
    probe = {}
    fwd = model.apply_model

    def rec(x_noisy, *a, **k):
        x_noisy.requires_grad_(True)
        probe["x"] = x_noisy
        return fwd(x_noisy, *a, **k)

    # the reference's training driver passes the pose map too; the stage-1 model ignores it
    cond = {"c_concat": [inp["pose"]], "c_crossattn": [inp["context"]], "image_control": [inp["ref"]], "wonoise": True}
    model.apply_model = rec
    try:
        with torch.enable_grad():
            model.train()
            loss, ld = model.p_losses(inp["x0"], cond, inp["t_train"], noise=inp["noise"])
            (loss * scale).backward()
    finally:
        del model.apply_model
    grads = {k: (None if p.grad is None else p.grad.detach().clone()) for k, p in model.named_parameters()
             if k.startswith(TRAINED)}
    return loss.detach(), ld, probe["x"].grad.detach().clone(), grads


def compare_grads(loss, dx, grads, tol):
    """worst errors against stage1_grad16.npz (grad16.npz's layout), each checked against tol[name]"""
    gold = G.load("stage1_grad16")
    names = [str(n) for n in gold["names"]]
    assert sorted(names) == sorted(grads)
    has = {n for n, h in zip(names, gold["has_grad"]) if h}
    assert {n for n in names if grads[n] is not None} == has  # has_grad exactly, time_embed included
    assert {n for n in has if n.startswith("model.diffusion_model.time_embed.")} == {
        f"model.diffusion_model.time_embed.{i}.{w}" for i in (0, 2) for w in ("weight", "bias")}
    worst = {"loss": abs(float(loss) - float(gold["loss"])) / float(gold["loss"]),
             "d_x_noisy": G.rel_l2(dx, torch.from_numpy(gold["d_x_noisy"])), "norm": 0.0, "sample": 0.0, "sum": 0.0,
             "full": 0.0}
    for i, n in enumerate(names):
        norm = float(gold["gnorm"][i])
        if grads[n] is None or norm == 0.0:
            continue
        g = grads[n].double().cpu().flatten()
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


def apply_inputs():
    return G.small32_inputs()


def chain_inputs():
    from magicdance_b200 import synth
    inp = synth.synth_inputs(1, 32, seed=5, shared_reference=True)
    uc_ctx = torch.randn(1, 77, 768, generator=torch.Generator().manual_seed(9))  # ignored by this branch
    c = {"c_concat": [inp["pose"]], "c_crossattn": [inp["context"]], "image_control": [inp["ref"]], "wonoise": True,
         "overlap_sampling": False}
    uc = {"c_concat": [inp["pose"]], "c_crossattn": [uc_ctx], "wonoise": True, "overlap_sampling": False}
    return inp, c, uc


def rename_for_stage2(sd):
    """load_state_dict_image_pose (train_tiktok.py:194-210): the stage-1 control_model becomes the appearance net"""
    return {k.replace("control_model", "appearance_control_model"): v for k, v in sd.items()}


def release_memory():
    """return freed host memory to the system: the CPU stand-ins leave gigabytes of small freed blocks in the heap,
    which the next test module's model could not otherwise reuse"""
    import ctypes
    import gc
    gc.collect()
    try:
        ctypes.CDLL("libc.so.6").malloc_trim(0)
    except (OSError, AttributeError):
        pass


@pytest.fixture(scope="module")
def model():
    m = stage1_model(freeze=False).eval()
    yield m
    del m
    release_memory()


@pytest.fixture
def fake_inference(monkeypatch):
    from magicdance_b200 import ops
    from tests import fake_ops
    from tests.test_engine_cpu import _PATCHED
    for name in _PATCHED + ("cfg_ddim_update",):
        monkeypatch.setattr(ops, name, getattr(fake_ops, name))
    prev = torch.is_grad_enabled()
    torch.set_grad_enabled(False)
    yield
    torch.set_grad_enabled(prev)


def test_yaml_targets_resolve_to_the_stage1_dropin_classes(model):
    import yaml
    from model_lib.ControlNet.cldm import cldm
    from magicdance_b200.dropin import cldm as dropin
    cfg = yaml.safe_load(open(YAML))["model"]
    assert cfg["target"] == "model_lib.ControlNet.cldm.cldm.ControlLDMReferenceOnly"
    assert cldm.ControlLDMReferenceOnly is dropin.ControlLDMReferenceOnly
    assert cldm.ControlledUnetModelAttn is dropin.ControlledUnetModelAttn
    assert type(model) is cldm.ControlLDMReferenceOnly
    assert type(model.model.diffusion_model) is cldm.ControlledUnetModelAttn
    assert type(model.control_model) is cldm.ControlNetReferenceOnly
    assert not hasattr(model, "pose_control_model") and not hasattr(model, "appearance_control_model")
    assert model.control_key == "hint" and model.only_mid_control is False
    assert model.channels == 4 and model.image_size == 64 and model.num_timesteps == 1000
    assert model.model.diffusion_model.use_checkpoint and model.control_model.use_checkpoint


def test_state_dict_keys_and_shapes_equal_the_reference(model):
    from magicdance_b200 import synth
    manifest = reference_manifest()  # recorded from the unmodified reference's stage-1 model, VAE included
    assert {k: list(v.shape) for k, v in model.state_dict().items()} == manifest
    assert any(k.startswith("control_model.input_hint_block.") for k in manifest)
    # a strict load of a checkpoint with exactly the reference's layout (load_state_dict_reference_only loads strictly)
    from model_lib.ControlNet.cldm.model import create_model
    m = create_model(YAML)
    missing, unexpected = m.load_state_dict({k: torch.zeros(v) for k, v in manifest.items()}, strict=True)
    assert not missing and not unexpected
    assert all(k in manifest for k in synth.SCHEDULE_KEYS)


def test_apply_model_and_bank_match_the_reference(model, fake_inference):
    g = G.load("stage1_32")
    inp = apply_inputs()
    cond = {"c_concat": [inp["pose"]], "c_crossattn": [inp["context"]]}
    eps_c = model.apply_model(inp["x"], inp["t"], cond, inp["ref"])
    eps_u = model.apply_model(inp["x"], inp["t"], {"c_crossattn": [inp["context"]]}, None, uc=True)
    e_c = G.rel_l2(eps_c, torch.from_numpy(g["apply/eps_c"]))
    e_u = G.rel_l2(eps_u, torch.from_numpy(g["apply/eps_u"]))
    assert e_c <= 5e-3 and e_u <= 5e-3, (e_c, e_u)
    # the sub-networks called on their own, as the reference's apply_model does (cldm.py:1071-1076)
    bank = []
    assert model.control_model(x=inp["ref"], hint=None, timesteps=inp["t"], context=inp["context"],
                               attention_bank=bank, attention_mode="write", uc=False) == []
    assert len(bank) == 16
    for i, b in enumerate(bank):
        G.check_summary(g, f"apply/bank{i}", b[0], 5e-3)
    residuals = [torch.ones(1)]  # ignored, and not consumed
    eps = model.model.diffusion_model(x=inp["x"], timesteps=inp["t"], context=inp["context"], control=bank,
                                      pose_control=residuals, only_mid_control=False, attention_mode="read", uc=False)
    assert torch.equal(eps, eps_c) and len(residuals) == 1
    plain = model.model.diffusion_model(x=inp["x"], timesteps=inp["t"], context=inp["context"], control=[],
                                        attention_mode="read", uc=True)
    assert torch.equal(plain, eps_u)
    assert model.engine().pose is None


def test_p_losses_forward_matches_the_reference(model, fake_inference):
    g = G.load("stage1_32")
    inp = apply_inputs()
    cond = {"c_concat": [inp["pose"]], "c_crossattn": [inp["context"]], "image_control": [inp["ref"]], "wonoise": True}
    out = {}
    fwd = model.apply_model

    def rec(*a, **k):
        out["eps"] = fwd(*a, **k)
        return out["eps"]

    model.apply_model = rec
    try:
        loss, ld = model.p_losses(torch.from_numpy(g["ploss/x0"]), cond, torch.from_numpy(g["ploss/t"]),
                                  noise=torch.from_numpy(g["ploss/noise"]))
    finally:
        del model.apply_model
    assert set(ld) == {"val/loss_simple", "val/loss_vlb", "val/loss"}
    assert G.rel_l2(out["eps"], torch.from_numpy(g["ploss/eps"])) <= 5e-3
    assert abs(float(loss) - float(g["ploss/loss"])) <= 1e-2 * float(g["ploss/loss"])
    assert abs(float(ld["val/loss_simple"]) - float(g["ploss/loss_simple"])) <= 1e-2 * float(g["ploss/loss_simple"])


def test_sample_log_four_step_chain_matches_the_reference(model, fake_inference):
    """sample_log -> DDIMSampler_ReferenceOnly.sample -> ddim_sampling -> p_sample_ddim, 'controlnet is more important'
    branch at CFG 7, against the reference sampler's own 4-step chain; no hint features are computed"""
    g = G.load("stage1_32")
    inp, c, uc = chain_inputs()
    model.image_size = 32
    try:
        x, inter = model.sample_log(c, 1, ddim=True, ddim_steps=4, eta=0.0, unconditional_guidance_scale=7.0,
                                    unconditional_conditioning=uc, x_T=inp["x"])
        pipe = next(iter(model._mdb_pipelines.values()))
        assert len(pipe._hint_cache) == 0 and len(pipe._bank_cache) == 4
    finally:
        model.image_size = 64
        model.__dict__.pop("_mdb_pipelines", None)
    assert G.rel_l2(x, torch.from_numpy(g["chain/x"])) <= 1e-2
    assert G.rel_l2(inter["pred_x0"][-1], torch.from_numpy(g["chain/pred_x0"])) <= 1e-2


def test_batched_cfg_branch_runs_without_a_pose_net(model, fake_inference):
    """ddim.py:539-566 (the unconditional conditioning keeps image_control): with no c_concat at all, the halves equal
    two separate conditional calls"""
    from magicdance_b200.dropin.ddim import DDIMSampler_ReferenceOnly
    inp, c, _ = chain_inputs()
    c = {k: v for k, v in c.items() if k != "c_concat"}
    uc = dict(c, c_crossattn=[torch.zeros(1, 77, 768)])
    s = DDIMSampler_ReferenceOnly(model)
    s.make_schedule(4, ddim_eta=0.0, verbose=False)
    t = torch.full((1,), int(s.ddim_timesteps[2]), dtype=torch.long)
    try:
        x_prev, _ = s.p_sample_ddim(inp["x"], c, t, index=2, unconditional_guidance_scale=7.0,
                                    unconditional_conditioning=uc)
    finally:
        model.__dict__.pop("_mdb_pipelines", None)
    e_c = model.apply_model(inp["x"], t, c, inp["ref"])
    e_u = model.apply_model(inp["x"], t, uc, inp["ref"])
    e = e_u + 7.0 * (e_c - e_u)
    a, ap = float(s.ddim_alphas[2]), float(s.ddim_alphas_prev[2])
    want = ap ** 0.5 * (inp["x"] - (1 - a) ** 0.5 * e) / a ** 0.5 + (1 - ap) ** 0.5 * e
    assert G.rel_l2(x_prev, want) <= 1e-2  # fp16 rounding differs between batch 2 and 1, CFG scales it


def test_a_stage1_checkpoint_renamed_for_stage2_writes_the_same_bank(model, fake_inference):
    """train_tiktok.py:194-210 loads the stage-1 checkpoint into the stage-2 model with control_model.* renamed to
    appearance_control_model.*: the appearance net then writes a bit-equal bank"""
    from model_lib.ControlNet.cldm.model import create_model
    s1 = model
    s2 = create_model(YAML_POSE)
    sd = rename_for_stage2(s1.state_dict())
    own = s2.state_dict()
    sd.update({k: torch.zeros_like(v) for k, v in own.items() if k.startswith("pose_control_model.")})
    missing, unexpected = s2.load_state_dict(sd, strict=True)
    assert not missing and not unexpected
    inp = apply_inputs()
    b1, b2 = [], []
    s1.control_model(x=inp["ref"], hint=None, timesteps=inp["t"], context=inp["context"], attention_bank=b1,
                     attention_mode="write")
    s2.appearance_control_model(x=inp["ref"], hint=None, timesteps=inp["t"], context=inp["context"], attention_bank=b2,
                                attention_mode="write")
    assert len(b1) == len(b2) == 16 and all(torch.equal(a[0], b[0]) for a, b in zip(b1, b2))
    del s2, sd, own, b1, b2
    release_memory()
