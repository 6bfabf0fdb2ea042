"""Stage-1 appearance-control pre-training (ControlLDMReferenceOnly) on the sm_90a kernels: the reference's stage-1
goldens (apply_model, bank, p_losses, a 4-step sample_log chain through the captured graphs, gradients), graph replay
against the eager loop, determinism of the training path, precision at 64x64 against the restatement's fp32 autograd,
inference after an optimizer step, and one training step at batch 32 (scripts/appearance_control_pretraining.sh)."""
import pytest
import torch

from oracle import restatement as R
from tests import golden_util as G
from tests.test_stage1_cpu import TOL, TRAINED, chain_inputs, compare_grads, stage1_model, train_step
from tests.test_train_gpu import _inputs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    m = stage1_model("cuda")
    yield m
    del m
    torch.cuda.empty_cache()


def _cuda(inp):
    return {k: v.cuda() for k, v in inp.items()}


def test_apply_model_bank_and_p_losses_match_the_reference(model):
    g = G.load("stage1_32")
    inp = _cuda(G.small32_inputs())
    cond = {"c_concat": [inp["pose"]], "c_crossattn": [inp["context"]]}
    with torch.no_grad():
        eps_c = model.apply_model(inp["x"], inp["t"], cond, inp["ref"])
        eps_u = model.apply_model(inp["x"], inp["t"], cond, None, uc=True)
        bank = []
        model.control_model(x=inp["ref"], hint=None, timesteps=inp["t"], context=inp["context"], attention_bank=bank,
                            attention_mode="write")
        model.eval()
        loss, ld = model.p_losses(torch.from_numpy(g["ploss/x0"]).cuda(), dict(cond, image_control=[inp["ref"]],
                                                                                 wonoise=True),
                                  torch.from_numpy(g["ploss/t"]).cuda(), noise=torch.from_numpy(g["ploss/noise"]).cuda())
        model.train()
    e = {"eps_c": G.rel_l2(eps_c, torch.from_numpy(g["apply/eps_c"])),
         "eps_u": G.rel_l2(eps_u, torch.from_numpy(g["apply/eps_u"])),
         "bank": max(G.check_summary(g, f"apply/bank{i}", b[0], 5e-3) for i, b in enumerate(bank)),
         "loss": abs(float(loss) - float(g["ploss/loss"])) / float(g["ploss/loss"])}
    print("stage-1 parity:", {k: f"{v:.3e}" for k, v in e.items()})
    assert len(bank) == 16 and e["eps_c"] <= 5e-3 and e["eps_u"] <= 5e-3 and e["loss"] <= 1e-2


def _sample_log(model, graphs):
    from magicdance_b200.dropin.ddim import DDIMSampler_ReferenceOnly
    inp, c, uc = chain_inputs()
    c, uc = ({k: [v[0].cuda()] if isinstance(v, list) else v for k, v in d.items()} for d in (c, uc))
    prev = DDIMSampler_ReferenceOnly.use_graphs
    DDIMSampler_ReferenceOnly.use_graphs = graphs
    model.image_size = 32
    try:
        with torch.no_grad():
            x, inter = model.sample_log(c, 1, ddim=True, ddim_steps=4, eta=0.0, unconditional_guidance_scale=7.0,
                                        unconditional_conditioning=uc, x_T=inp["x"].cuda())
    finally:
        DDIMSampler_ReferenceOnly.use_graphs = prev
        model.image_size = 64
    return x, inter["pred_x0"][-1]


def test_sample_log_replays_the_graphs_and_matches_the_reference(model):
    """train_tiktok.py:437-444 logs samples through sample_log: the stage-1 chain replays the captured step and bank
    graphs (no hint buffer, no side stream, no pose time table) and matches the reference chain and the eager loop"""
    from magicdance_b200 import ops
    g = G.load("stage1_32")
    n0 = ops.launch_count()
    x, p0 = _sample_log(model, graphs=True)
    ents = list(model._mdb_graphs.values())
    assert len(ents) == 1
    gd = ents[0]["gd"]
    assert gd.replayed_launches > 0 and gd.hint is None and gd.side is None and gd.emb_pose is None
    assert gd.step_launches > 0 and gd.step_launches < 512
    x_e, p0_e = _sample_log(model, graphs=False)
    e = {"x": G.rel_l2(x, torch.from_numpy(g["chain/x"])), "pred_x0": G.rel_l2(p0, torch.from_numpy(g["chain/pred_x0"])),
         "graph_vs_eager": G.rel_l2(x, x_e)}
    print(f"stage-1 chain: {e}, step graph {gd.step_launches} launches, bank graph {gd.bank_launches}; "
          f"{ops.launch_count() - n0} launches counted")
    assert e["x"] <= 1e-2 and e["pred_x0"] <= 1e-2 and e["graph_vs_eager"] <= 5e-3
    model.__dict__.pop("_mdb_graphs", None)
    model.__dict__.pop("_mdb_pipelines", None)


def test_eager_sampler_branches_run_without_a_pose_net(model):
    """batched CFG, eta != 0 and a noised reference take the eager step; all stay finite and need no c_concat"""
    from model_lib.ControlNet.ldm.models.diffusion.ddim import DDIMSampler_ReferenceOnly
    inp, c, _ = chain_inputs()
    c = {"c_crossattn": [inp["context"].cuda()], "image_control": [inp["ref"].cuda()], "wonoise": True}
    s = DDIMSampler_ReferenceOnly(model)
    s.make_schedule(4, ddim_eta=0.0, verbose=False)
    t = torch.full((1,), int(s.ddim_timesteps[2]), dtype=torch.long, device="cuda")
    x = inp["x"].cuda()
    with torch.no_grad():
        outs = [s.p_sample_ddim(x, c, t, index=2, unconditional_guidance_scale=7.0,
                                unconditional_conditioning=dict(c, c_crossattn=[torch.zeros_like(inp["context"]).cuda()]))[0],
                s.p_sample_ddim(x, dict(c, wonoise=False), t, index=2, unconditional_guidance_scale=7.0,
                                unconditional_conditioning={"c_crossattn": c["c_crossattn"]})[0]]
        s.make_schedule(4, ddim_eta=0.5, verbose=False)
        outs.append(s.p_sample_ddim(x, c, t, index=2, unconditional_guidance_scale=7.0,
                                    unconditional_conditioning={"c_crossattn": c["c_crossattn"]})[0])
    assert all(o.shape == x.shape and torch.isfinite(o).all() for o in outs)
    model.__dict__.pop("_mdb_pipelines", None)


def test_grad16_parity_with_the_reference(model):
    loss, ld, dx, grads = train_step(model)
    assert set(ld) == {"train/loss_simple", "train/loss_vlb", "train/loss"}
    print("stage-1 grad16 worst:", compare_grads(loss, dx, grads, TOL))


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
    """latent 64x64, B = 1, against the restatement's fp32 autograd of the stage-1 forward (appearance 'write' pass,
    UNet in 'read' mode without residuals): every reached gradient within 2e-2 rel-L2, d_x_noisy within 1e-2, the
    loss within 5e-3; then the same under a x65536 loss scale"""
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        inp = _inputs(1, 64, seed=41)
        loss, _, dx, grads = train_step(model, inp)
        reached = [k for k, g in grads.items() if g is not None and float(g.abs().max()) > 0]
        sd = {k: v.detach().clone().requires_grad_(k.startswith(TRAINED)) for k, v in model.state_dict().items()
              if v.is_floating_point()}
        dev = _cuda(inp)
        x_noisy = R.q_sample(dev["x0"], dev["t_train"], dev["noise"], R.make_schedule()["alphas_cumprod"]).requires_grad_()
        with torch.enable_grad():
            bank = R.appearance_forward(sd, "control_model.", dev["ref"], dev["t_train"], dev["context"])
            eps = R.unet_forward(sd, R.UNET, x_noisy, dev["t_train"], dev["context"], bank=bank)
            rl = ((eps - dev["noise"]) ** 2).mean()
            rl.backward()
        ref = {k: sd[k].grad for k in reached}
        rdx = x_noisy.grad
        del sd, bank, eps
        errs = {k: G.rel_l2(grads[k], ref[k]) for k in reached}
        worst = max(errs, key=errs.get)
        e_dx = G.rel_l2(dx, rdx)
        print(f"stage-1 64x64: loss {float(loss):.6f} vs {float(rl):.6f}; d_x_noisy {e_dx:.3e}; worst parameter {worst} "
              f"{errs[worst]:.3e}; time_embed {max(v for k, v in errs.items() if k.startswith(TRAINED[1])):.3e}")
        assert abs(float(loss) - float(rl)) <= 5e-3 * float(rl)
        assert e_dx <= 1e-2 and errs[worst] <= 2e-2
        assert any(k.startswith(TRAINED[1]) for k in reached)
        S = 65536.0
        _, _, sdx, sgrads = train_step(model, inp, scale=S)
        serrs = {k: G.rel_l2(sgrads[k] / S, ref[k]) for k in reached}
        print(f"stage-1 64x64 with a x{S:g} loss scale: d_x_noisy {G.rel_l2(sdx / S, rdx):.3e}; worst parameter "
              f"{max(serrs.values()):.3e}")
        assert G.rel_l2(sdx / S, rdx) <= 1e-2 and max(serrs.values()) <= 2e-2
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32


def _eps(m, inp):
    dev = _cuda(inp)
    with torch.no_grad():
        return m.apply_model(dev["x"], dev["t_train"], {"c_crossattn": [dev["context"]]}, dev["ref"])


def test_inference_after_training_sees_the_new_weights(model):
    inp = _inputs(2, 32, seed=7)
    before = _eps(model, inp)
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-3)
    train_step(model)
    opt.step()
    after = _eps(model, inp)
    assert not torch.equal(after, before)
    fresh = stage1_model("cpu")
    fresh.load_state_dict(model.state_dict())
    fresh = fresh.cuda()
    assert torch.equal(after, _eps(fresh, inp))
    del fresh, opt
    model.load_state_dict(stage1_model("cpu").state_dict())  # the weights the other tests expect
    model.zero_grad(set_to_none=True)


def test_batch32_step_runs_with_finite_gradients():
    """scripts/appearance_control_pretraining.sh: --train_batch_size 32 on one GPU, 64x64 latent, checkpointing, AdamW"""
    m = stage1_model("cuda")
    opt = torch.optim.AdamW([p for p in m.parameters() if p.requires_grad], lr=1e-5)
    torch.cuda.reset_peak_memory_stats()
    loss, _, dx, grads = train_step(m, _inputs(32, 64, seed=3))
    opt.step()
    torch.cuda.synchronize()
    print(f"stage-1 batch 32 step: loss {float(loss):.5f}, peak allocated {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
    assert torch.isfinite(loss) and torch.isfinite(dx).all()
    assert all(torch.isfinite(g).all() for g in grads.values() if g is not None)
    assert all(torch.isfinite(p).all() for p in m.parameters() if p.requires_grad)
    del m, opt
    torch.cuda.empty_cache()
