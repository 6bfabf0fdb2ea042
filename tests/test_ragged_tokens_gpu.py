"""Sampling on the GPU at latents whose attention levels hold a number of tokens that is not a multiple of 8 (40x24:
60 tokens at level 2 and 15 in the middle block; 48x48 and 80x80: 36 and 100 in the middle block).  Self-attention V^T, the
bank's V^T and the bank slots are laid out with each sample's columns padded to a multiple of 8 (ops.pad_tokens); the
kernels never read the padding.  Checked against the unmodified reference's golden at 40x24, the CPU restatement at
48x48 and 80x80, eager steps against graph replay, and the 64x64 step graph's launch counts."""
import pytest
import torch

from magicdance_b200 import ops
from oracle import restatement as R
from tests import golden_util as G
from tests.test_train_cpu import stage2_model

pytestmark = pytest.mark.gpu

_PAD_TOKENS = ops.pad_tokens


@pytest.fixture(autouse=True)
def no_im2col_buffer(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("im2col3x3 launched for a UNet conv")

    monkeypatch.setattr(ops, "im2col3x3", refuse)


@pytest.fixture(scope="module")
def model():
    m = stage2_model("cuda").eval()
    yield m
    del m
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def engine():
    from magicdance_b200 import synth
    from magicdance_b200.engine import DenoiseEngine
    eng = DenoiseEngine(synth.synth_state_dict(seed=0), device="cuda")
    yield eng
    del eng
    torch.cuda.empty_cache()


def _inputs(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    pose = (torch.rand(b, 3, 8 * h, 8 * w, generator=g) > 0.97).float() * torch.rand(b, 3, 8 * h, 8 * w, generator=g)
    return {"x": torch.randn(b, 4, h, w, generator=g), "ref": 0.8 * torch.randn(b, 4, h, w, generator=g), "pose": pose,
            "context": torch.randn(b, 77, 768, generator=g), "uc_context": torch.randn(1, 77, 768, generator=g)}


def _chain(model, shape, x_T, c, uc, graphs):
    from magicdance_b200.dropin.ddim import DDIMSampler_ReferenceOnly
    sampler = DDIMSampler_ReferenceOnly(model)
    sampler.use_graphs = graphs
    with torch.no_grad():
        x, inter = sampler.sample(4, x_T.shape[0], shape, c, verbose=False, eta=0.0, x_T=x_T,
                                  unconditional_guidance_scale=7.0, unconditional_conditioning=uc)
    return x, inter["pred_x0"][-1]


def _forget_graphs(model):
    model.__dict__.pop("_mdb_graphs", None)
    model.__dict__.pop("_mdb_pipelines", None)
    torch.cuda.empty_cache()


def test_apply_model_at_40x24_matches_the_reference_golden(model):
    """B = 2, per-sample t and reference latent, conditional and uc=True"""
    from tests import anysize_golden as A
    gold, inp = A.load()
    inp = {k: v.cuda() for k, v in inp.items()}
    cond = {"c_concat": [inp["pose"]], "c_crossattn": [inp["context"]]}
    with torch.no_grad():
        eps_c = model.apply_model(inp["x"], inp["t"], cond, inp["ref"])
        eps_u = model.apply_model(inp["x"], inp["t"], cond, None, uc=True)
    e_c = G.rel_l2(eps_c, torch.from_numpy(gold["apply/eps_c"]))
    e_u = G.rel_l2(eps_u, torch.from_numpy(gold["apply/eps_u"]))
    print(f"40x24 eps rel-L2: cond {e_c:.3e}, uncond {e_u:.3e}")
    assert e_c <= 5e-3 and e_u <= 5e-3


def test_sampler_chain_at_40x24_replays_the_graphs(model):
    """the drop-in sampler's 4-step chain at CFG 7 (what sample_log runs) takes the graphed path at 40x24 and matches
    the reference's chain; two graphed runs are bit-equal and the eager loop agrees"""
    from tests import anysize_golden as A
    gold, inp = A.load()
    inp = {k: v.cuda() for k, v in inp.items()}
    c = {"c_concat": [inp["pose"][:1]], "c_crossattn": [inp["context"][:1]], "image_control": [inp["ref"][:1]],
         "wonoise": True, "overlap_sampling": False}
    uc = {"c_concat": [inp["pose"][:1]], "c_crossattn": [inp["uc_context"]], "wonoise": True, "overlap_sampling": False}
    try:
        x, p0 = _chain(model, (4, 40, 24), inp["x"][:1], c, uc, graphs=True)
        assert len(model.__dict__.get("_mdb_graphs", {})) == 1  # the graphed path was taken
        x2, p02 = _chain(model, (4, 40, 24), inp["x"][:1], c, uc, graphs=True)
        x_e, _ = _chain(model, (4, 40, 24), inp["x"][:1], c, uc, graphs=False)
    finally:
        _forget_graphs(model)
    e = {"x": G.rel_l2(x, torch.from_numpy(gold["chain/x"])),
         "pred_x0": G.rel_l2(p0, torch.from_numpy(gold["chain/pred_x0"])), "graph_vs_eager": G.rel_l2(x, x_e)}
    print(f"40x24 chain: {e}")
    assert e["x"] <= 1e-2 and e["pred_x0"] <= 1e-2 and e["graph_vs_eager"] <= 2e-3
    assert torch.equal(x, x2) and torch.equal(p0, p02)


@pytest.mark.parametrize("side", [48, 80])
def test_eps_matches_the_restatement(engine, side):
    from magicdance_b200 import synth
    inp = _inputs(1, side, side, seed=side)
    t = torch.tensor([621])
    with torch.no_grad():
        e_gpu = engine.apply_model(inp["x"].cuda(), t.cuda(), inp["context"].cuda(), inp["pose"].cuda(),
                                   inp["ref"].cuda(), uc=False)
        e_ref = R.apply_model(synth.synth_state_dict(seed=0), inp["x"], t, inp["context"], inp["pose"], inp["ref"],
                              uc=False)
    err = G.rel_l2(e_gpu, e_ref)
    print(f"{side}x{side} eps rel-L2 vs restatement {err:.3e}")
    assert err <= 5e-3


def test_eight_frames_graphed_match_eager_steps_at_80x80(engine):
    """GraphedDenoiser with 8 frames at 80x80 (step graph + timestep-batched bank graph into padded slots) against
    DenoisePipeline.step over a 3-step chain"""
    from magicdance_b200.pipeline import DenoisePipeline, GraphedDenoiser
    inp = {k: v.cuda() for k, v in _inputs(8, 80, 80, seed=80).items()}
    ctx = inp["context"][:1].contiguous()
    ref = inp["ref"][:1].contiguous()
    pipe = DenoisePipeline(engine)
    hint = pipe.hint(inp["pose"])
    idxs = [49, 48, 47]
    with torch.no_grad():
        gd = GraphedDenoiser(pipe, 8, (80, 80), ctx, bank_chunk=4).capture()
        slots = torch.zeros((3, gd.layout.numel), dtype=torch.float16, device="cuda")
        gd.build_bank(idxs, ref, slots)
        gd.hint.copy_(hint)
        gd.x.copy_(inp["x"])
        x_e = inp["x"]
        for j, ix in enumerate(idxs):
            x_e, _, _, _ = pipe.step(x_e, ix, ctx, hint, pipe.reference_bank(ref, ctx, ix))
            x_g = gd.step(ix, slots[j]).clone()
            err = G.rel_l2(x_g, x_e)
            print(f"80x80, 8 frames, step {j}: graph vs eager {err:.3e}")
            assert err <= 2e-3
    assert torch.isfinite(x_g).all()
    del gd
    pipe.clear_caches()
    torch.cuda.empty_cache()


def test_stage1_graph_replay_matches_eager_at_48x48():
    """the stage-1 ControlLDMReferenceOnly (no pose net) at 48x48: the drop-in sampler's graph replay against its
    eager loop"""
    from tests.test_stage1_cpu import stage1_model
    m = stage1_model("cuda").eval()
    inp = {k: v.cuda() for k, v in _inputs(1, 48, 48, seed=148).items()}
    c = {"c_concat": [inp["pose"]], "c_crossattn": [inp["context"]], "image_control": [inp["ref"]], "wonoise": True,
         "overlap_sampling": False}
    uc = {"c_concat": [inp["pose"]], "c_crossattn": [inp["uc_context"]], "wonoise": True, "overlap_sampling": False}
    try:
        x, _ = _chain(m, (4, 48, 48), inp["x"], c, uc, graphs=True)
        assert len(m.__dict__.get("_mdb_graphs", {})) == 1
        x_e, _ = _chain(m, (4, 48, 48), inp["x"], c, uc, graphs=False)
    finally:
        _forget_graphs(m)
        del m
        torch.cuda.empty_cache()
    err = G.rel_l2(x, x_e)
    print(f"stage 1, 48x48 chain: graph vs eager {err:.3e}")
    assert torch.isfinite(x).all() and err <= 5e-3


def _nan_padding(x, b):
    """ops.pad_tokens with the padding rows set to NaN (so are the V^T columns projected from them)"""
    xp, ldv = _PAD_TOKENS(x, b)
    if xp is not x:
        xp.view(b, ldv, -1)[:, x.shape[0] // b:] = float("nan")
    return xp, ldv


def test_padding_is_never_read_at_40x24(engine, monkeypatch):
    """padded token rows and V^T padding columns (self-attention, bank, bank slots and text) filled with NaN: eps and
    a graphed step are bit-equal to the runs with zero padding"""
    from magicdance_b200.pipeline import DenoisePipeline, GraphedDenoiser
    from tests import anysize_golden as A
    _, inp = A.load()
    inp = {k: v.cuda() for k, v in inp.items()}
    out = []
    for pad in (ops.pad_tokens, _nan_padding):
        monkeypatch.setattr(ops, "pad_tokens", pad)
        engine._ctx_cache.clear()
        with torch.no_grad():
            eps = engine.apply_model(inp["x"], inp["t"], inp["context"], inp["pose"], inp["ref"], uc=False)
            pipe = DenoisePipeline(engine)
            gd = GraphedDenoiser(pipe, 1, (40, 24), inp["context"][:1].contiguous(), bank_chunk=2).capture()
            slots = torch.zeros((1, gd.layout.numel), dtype=torch.float16, device="cuda")
            gd.build_bank([49], inp["ref"][:1], slots)
            gd.hint.copy_(pipe.hint(inp["pose"][:1]))
            gd.x.copy_(inp["x"][:1])
            x = gd.step(49, slots[0]).clone()
        out.append((eps, x, slots))
        del gd
    engine._ctx_cache.clear()
    torch.cuda.empty_cache()
    assert torch.isnan(out[1][2].float()).any()  # the NaN padding did reach the bank slot
    assert torch.isfinite(out[0][0]).all() and torch.isfinite(out[0][1]).all()
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


@pytest.mark.parametrize("frames,launches", [(1, 512), (8, 533)])
def test_step_graph_launches_unchanged_at_64x64(engine, frames, launches):
    """at 64x64 every level has a multiple of 8 tokens: no padding copy, and the step graph holds the same library
    launches as before"""
    from magicdance_b200.pipeline import DenoisePipeline, GraphedDenoiser
    copied = []  # token counts of the pad_tokens calls that copied

    def recording(x, b):
        xp, ldv = real(x, b)
        if xp is not x:
            copied.append(x.shape[0] // b)
        return xp, ldv

    real = ops.pad_tokens
    monkeypatch = pytest.MonkeyPatch()
    monkeypatch.setattr(ops, "pad_tokens", recording)
    try:
        ctx = torch.randn(1, 77, 768, device="cuda")
        with torch.no_grad():
            gd = GraphedDenoiser(DenoisePipeline(engine), frames, (64, 64), ctx, bank_chunk=2).capture()
    finally:
        monkeypatch.undo()
    print(f"64x64, {frames} frame(s): {gd.step_launches} launches per step")
    assert gd.step_launches == launches
    assert set(copied) <= {77}  # only the text tokens (77 -> 80), once per context
    del gd
    engine._ctx_cache.clear()
    torch.cuda.empty_cache()
