"""Sampling at latents whose attention levels hold a number of tokens that is not a multiple of 8 (40x24: 60 tokens at
level 2 and 15 in the middle block; 48x48: 36 in the middle block), on CPU stand-ins that enforce the C ABI's alignment rules:
every V^T column block of one sample starts 16-byte aligned (ldv*_batch % 8 == 0), and so does every GEMM output row.
The plain stand-ins of tests/fake_ops.py compute the same numbers without those checks, so they cannot tell whether
the engine's operands would be accepted by the kernels.  Also the padded bank layout (parallel.BankLayout) and its
exchange over gloo."""
import gc
from types import SimpleNamespace

import pytest
import torch

from tests import fake_ops
from tests import golden_util as G


def _aligned(t):
    return t.stride(-1) == 1 and t.stride(0) % 8 == 0 and t.data_ptr() % 16 == 0


def strict_gemm(a, w, *, out=None, **kw):
    """tests/fake_ops.gemm behind mdb_gemm_f16's output check: D's rows 16-byte aligned (ldd % 8 == 0)"""
    n_out = w.shape[0] // 2 if kw.get("epilogue") == 1 else w.shape[0]
    if out is not None:
        assert _aligned(out), ("gemm: D must have ldd % 8 == 0 and be 16-byte aligned", tuple(out.shape), out.stride())
    else:  # ops.gemm allocates D as a contiguous [M, N]: ldd = N
        assert n_out % 8 == 0, f"gemm: ldd = N = {n_out} must be a multiple of 8"
    return fake_ops.gemm(a, w, out=out, **kw)


def strict_attention(q, k0, vt0, n0, *, heads, d, batch, nq, kv0_batches=None, ldv0_batch=None, k1=None, vt1=None,
                     n1=0, kv1_batches=1, ldv1_batch=None, bank_batches=0, **kw):
    """tests/fake_ops.attention behind mdb_attention_f16's operand checks (attention_check_desc, tmap_vt)"""
    ldv0 = n0 if ldv0_batch is None else ldv0_batch
    kvb0 = batch if kv0_batches is None else kv0_batches
    assert ldv0 >= n0 and ldv0 % 8 == 0, f"attention: ldv0_batch = {ldv0} must be >= n0 = {n0} and a multiple of 8"
    assert _aligned(vt0), ("attention: V^T row stride", tuple(vt0.shape), vt0.stride())
    assert vt0.shape[1] >= (kvb0 - 1) * ldv0 + n0
    if n1:
        ldv1 = n1 if ldv1_batch is None else ldv1_batch
        assert ldv1 >= n1 and ldv1 % 8 == 0, f"attention: ldv1_batch = {ldv1} must be >= n1 = {n1} and a multiple of 8"
        assert _aligned(vt1), ("attention: bank V^T row stride", tuple(vt1.shape), vt1.stride())
        assert vt1.shape[1] >= (kv1_batches - 1) * ldv1 + n1
    return fake_ops.attention(q, k0, vt0, n0, heads=heads, d=d, batch=batch, nq=nq, kv0_batches=kv0_batches,
                              ldv0_batch=ldv0_batch, k1=k1, vt1=vt1, n1=n1, kv1_batches=kv1_batches,
                              ldv1_batch=ldv1_batch, bank_batches=bank_batches, **kw)


@pytest.fixture(scope="module")
def strict_model():
    """the stage-2 drop-in model with every kernel entry point of inference on the stand-ins, GEMM and attention
    behind the C ABI's alignment checks"""
    from magicdance_b200 import ops
    from tests import fake_igemm_ops
    from tests.test_engine_cpu import _PATCHED
    from tests.test_train_cpu import stage2_model

    def refuse(*a, **k):
        raise AssertionError("im2col3x3 called for a UNet conv")

    with pytest.MonkeyPatch.context() as mp, torch.no_grad():
        for name in _PATCHED + ("cfg_ddim_update",):
            mp.setattr(ops, name, getattr(fake_ops, name))
        mp.setattr(ops, "gemm", strict_gemm)
        mp.setattr(ops, "attention", strict_attention)
        mp.setattr(ops, "im2col3x3", refuse)
        mp.setattr(ops, "conv3x3_igemm", fake_igemm_ops.conv3x3_igemm)
        model = stage2_model().eval()
        yield model
        del model
        gc.collect()


def test_apply_model_at_40x24_on_strict_stand_ins(strict_model):
    """apply_model at 40x24, B = 2, per-sample t and reference, conditional and uc=True, against the reference's eps"""
    from tests import anysize_golden as A
    gold, inp = A.load()
    cond = {"c_concat": [inp["pose"]], "c_crossattn": [inp["context"]]}
    eps_c = strict_model.apply_model(inp["x"], inp["t"], cond, inp["ref"])
    eps_u = strict_model.apply_model(inp["x"], inp["t"], cond, None, uc=True)
    e_c = G.rel_l2(eps_c, torch.from_numpy(gold["apply/eps_c"]))
    e_u = G.rel_l2(eps_u, torch.from_numpy(gold["apply/eps_u"]))
    print(f"40x24 eps rel-L2 (strict stand-ins): cond {e_c:.3e}, uncond {e_u:.3e}")
    assert e_c <= 5e-3 and e_u <= 5e-3


def test_sampler_chain_at_40x24_on_strict_stand_ins(strict_model):
    """the drop-in DDIMSampler_ReferenceOnly.sample, 4 DDIM steps at CFG 7 with a (4, 40, 24) shape (B = 1: 15 tokens
    in the middle block, so V^T of one sample is 15 columns wide unless padded)"""
    from magicdance_b200.dropin.ddim import DDIMSampler_ReferenceOnly
    from tests import anysize_golden as A
    gold, inp = A.load()
    c = {"c_concat": [inp["pose"][:1]], "c_crossattn": [inp["context"][:1]], "image_control": [inp["ref"][:1]],
         "wonoise": True, "overlap_sampling": False}
    uc = {"c_concat": [inp["pose"][:1]], "c_crossattn": [inp["uc_context"]], "wonoise": True, "overlap_sampling": False}
    try:
        x, inter = DDIMSampler_ReferenceOnly(strict_model).sample(
            4, 1, (4, 40, 24), c, verbose=False, eta=0.0, x_T=inp["x"][:1], unconditional_guidance_scale=7.0,
            unconditional_conditioning=uc)
    finally:
        strict_model.__dict__.pop("_mdb_pipelines", None)
    e_x = G.rel_l2(x, torch.from_numpy(gold["chain/x"]))
    e_p = G.rel_l2(inter["pred_x0"][-1], torch.from_numpy(gold["chain/pred_x0"]))
    print(f"40x24 4-step chain rel-L2 (strict stand-ins): x {e_x:.3e}, pred_x0 {e_p:.3e}")
    assert e_x <= 1e-2 and e_p <= 1e-2


def test_apply_model_at_48x48_on_strict_stand_ins_matches_the_oracle(strict_model):
    """48x48, B = 1 (36 tokens in the middle block) against the CPU restatement"""
    from magicdance_b200 import synth
    from oracle import restatement as R
    g = torch.Generator().manual_seed(48)
    x = torch.randn(1, 4, 48, 48, generator=g)
    ref = 0.8 * torch.randn(1, 4, 48, 48, generator=g)
    pose = (torch.rand(1, 3, 384, 384, generator=g) > 0.97).float() * torch.rand(1, 3, 384, 384, generator=g)
    ctx = torch.randn(1, 77, 768, generator=g)
    t = torch.tensor([621])
    eps = strict_model.apply_model(x, t, {"c_concat": [pose], "c_crossattn": [ctx]}, ref)
    sd = synth.synth_state_dict(seed=0)
    with torch.no_grad():
        e_ref = R.apply_model(sd, x, t, ctx, pose, ref, uc=False)
    del sd
    gc.collect()
    err = G.rel_l2(eps, e_ref)
    print(f"48x48 eps rel-L2 (strict stand-ins) vs restatement: {err:.3e}")
    assert err <= 5e-3


def _geometry(h, w):
    """(tokens, channels) of the 16 attention layers for an h x w latent: engine.attn_geometry over the block plan"""
    from magicdance_b200.engine import DenoiseEngine, NetConfig, block_plan
    eng = DenoiseEngine.__new__(DenoiseEngine)
    eng.unet = SimpleNamespace(**dict(zip(("inp", "mid", "out"), block_plan(NetConfig()))))
    return eng.attn_geometry(h, w)


def test_bank_layout_pads_v_transposed_at_40x24():
    from magicdance_b200 import parallel
    geo = _geometry(40, 24)
    assert sorted({n for n, _ in geo}) == [15, 60, 240, 960]
    layout = parallel.BankLayout(geo)
    flat = torch.zeros(layout.numel, dtype=torch.float16)
    views = layout.views(flat, [n for n, _ in geo], 1)
    end = 0
    for (n, c), off, (k, vt, n_, b) in zip(geo, layout.offsets, views):
        ldv = (n + 7) // 8 * 8
        assert (n_, b) == (n, 1) and k.shape == (n, c) and vt.shape == (c, ldv)
        assert off % 8 == 0 and (off + n * c) % 8 == 0  # K and V^T blocks start 16-byte aligned
        assert k.data_ptr() == flat.data_ptr() + 2 * off and vt.data_ptr() == k.data_ptr() + 2 * n * c
        assert off == end  # contiguous, in bank order
        end = off + n * c + c * ldv
    assert layout.numel == (end + 127) // 128 * 128 and layout.numel % 128 == 0


def test_bank_layout_is_unchanged_where_every_level_tiles():
    """at 64x64 every layer's token count is a multiple of 8: the layout (what the all-gather moves) is the unpadded
    K [N, C] + V^T [C, N] per layer"""
    from magicdance_b200 import parallel
    geo = _geometry(64, 64)
    layout = parallel.BankLayout(geo)
    off, offsets = 0, []
    for n, c in geo:
        offsets.append(off)
        off += 2 * n * c
    assert layout.offsets == offsets and layout.numel == (off + 127) // 128 * 128
    for (n, c), (_, vt, _, _) in zip(geo, layout.views(torch.zeros(layout.numel, dtype=torch.float16),
                                                       [n for n, _ in geo], 1)):
        assert vt.shape == (c, n)


def test_project_bank_and_slots_carry_the_padded_v_transposed():
    """project_bank's V^T of a ragged layer is [C, batches*ldv], and build_bank_slots copies each timestep's [C, ldv]
    into its slot: a slot's views equal the directly projected bank, padding columns excluded"""
    from magicdance_b200 import ops, parallel
    from magicdance_b200.engine import DenoiseEngine
    from magicdance_b200.pipeline import build_bank_slots
    torch.manual_seed(0)
    c, n, tb = 64, 15, 3
    a = type("A", (), {})()
    a.c = c
    a.wqk = torch.randn(2 * c, c).half()
    a.wv = torch.randn(c, c).half()
    eng = DenoiseEngine.__new__(DenoiseEngine)
    eng.unet = type("N", (), {"attn_layers": lambda self: [a]})()
    bank = [torch.randn(tb * n, c).half()]
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ops, "gemm", strict_gemm)
        (k, vt, n_, b), = eng.project_bank(bank, tb)
        assert (n_, b) == (n, tb) and k.shape == (tb * n, c) and vt.shape == (c, tb * 16)
        layout = parallel.BankLayout([(n, c)])
        slots = torch.zeros((tb, layout.numel), dtype=torch.float16)
        eng.bank_kv = lambda ref, t, ctx: eng.project_bank(bank, tb)
        build_bank_slots(eng, torch.zeros(1, 4, 8, 8), torch.zeros(tb, dtype=torch.long), torch.zeros(1, 77, 768),
                         layout, [n], slots)
    for j in range(tb):
        (ks, vts, _, _), = layout.views(slots[j], [n], 1)
        assert torch.equal(ks, k[j * n:(j + 1) * n])
        assert torch.equal(vts[:, :n], vt[:, j * 16:j * 16 + n])
        assert torch.equal(vts[:, :n], (bank[0][j * n:(j + 1) * n].float() @ a.wv.float().t()).t().half())


def test_pad_tokens():
    from magicdance_b200 import ops
    x = torch.randn(2 * 64, 32)
    assert ops.pad_tokens(x, 2) == (x, 64) and ops.pad_tokens(x, 2)[0] is x  # no copy where n % 8 == 0
    x = torch.randn(2 * 15, 32, requires_grad=True)
    with torch.enable_grad():
        xp, ldv = ops.pad_tokens(x, 2)
        xp.sum().backward()  # differentiable: the padding rows get no gradient to pass on
    assert ldv == 16 and xp.shape == (32, 32)
    assert torch.equal(xp[:15], x[:15]) and torch.equal(xp[16:31], x[15:]) and not xp[15].any() and not xp[31].any()
    assert torch.equal(x.grad, torch.ones_like(x))


# ---------------------------------------------------------------------------------------------------------------------
# the bank exchange with the 40x24 layout (tests/test_parallel_gloo.py's harness)
# ---------------------------------------------------------------------------------------------------------------------
def _exchange_worker(rank, world, port, q):
    import os

    import torch.distributed as dist

    from magicdance_b200 import parallel as P
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    geo = _geometry(40, 24)
    tokens = [n for n, _ in geo]
    layout = P.BankLayout(geo)

    def value(index, li, shape, sign):
        return sign * (index + 0.25 * li + torch.arange(shape[0] * shape[1]).reshape(shape) % 7)

    def build_fn(chunk, slots):
        for index, flat in zip(chunk, slots):
            for li, (k, vt, n, b) in enumerate(layout.views(flat, tokens, 1)):
                k.copy_(value(index, li, k.shape, 1))
                vt.copy_(value(index, li, vt.shape, -1))

    indices = list(range(9, -1, -1))
    table = P.build_and_gather_bank(indices, layout, build_fn, "cpu", world, rank, chunk=3)
    table.wait()
    ok = sorted(table) == list(range(10))
    for ix, flat in table.items():
        for li, (k, vt, n, b) in enumerate(layout.views(flat, tokens, 1)):
            ok &= torch.equal(k, value(ix, li, k.shape, 1).half()) and torch.equal(vt, value(ix, li, vt.shape, -1).half())
    everything = torch.stack([table[ix] for ix in range(10)])
    gathered = [torch.zeros_like(everything) for _ in range(world)]
    dist.all_gather(gathered, everything)
    ok &= all(torch.equal(g, gathered[0]) for g in gathered)  # every rank ends with identical slots
    q.put((rank, bool(ok)))
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_bank_exchange_at_40x24_gloo(world):
    import torch.multiprocessing as mp

    from tests.test_parallel_gloo import _free_port
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_exchange_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
    assert [r[1] for r in res] == [True] * world
