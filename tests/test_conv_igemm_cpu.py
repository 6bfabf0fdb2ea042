"""CPU-only checks of the 3x3 convolution at any latent size: its C ABI (descriptors, compiled resources, argument
refusal before any launch), the training forward's latent-size rule, and the orchestration at 40x24 (a latent where no
level tiles into the box path's TMA boxes) on CPU stand-ins (tests/fake_igemm_ops.py, tests/fake_ops.py,
tests/fake_train_ops.py) against the unmodified reference's golden (tests/golden/anysize40x24.npz): gradients, eps and a
4-step sampler chain."""
import ctypes as C
import os
import re

import pytest
import torch

from tests.test_attention_bwd_cpu import _kernels

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_new_entry_points_take_the_gemm_descriptors():
    """mdb_conv3x3_igemm_* use mdb_gemm_desc / mdb_gemm_bwd_desc unchanged (their mirrors are checked against the
    header by tests/test_gemm_bwd_cpu.py): no new descriptor, no new struct id"""
    from magicdance_b200 import _lib
    with open(os.path.join(REPO, "include", "magicdance_b200.h")) as f:
        hdr = f.read()
    assert "int mdb_conv3x3_igemm_f16(const mdb_gemm_desc* desc, mdb_stream_t stream);" in hdr
    assert "int mdb_conv3x3_igemm_bwd_f16(const mdb_gemm_bwd_desc* desc, mdb_stream_t stream);" in hdr
    assert "int64_t mdb_conv3x3_igemm_bwd_ws_floats(const mdb_gemm_bwd_desc* desc);" in hdr
    sig = _lib.SIGNATURES
    assert sig["mdb_conv3x3_igemm_f16"][1][0]._type_ is _lib.GemmDesc
    assert sig["mdb_conv3x3_igemm_bwd_f16"][1][0]._type_ is _lib.GemmBwdDesc
    lib = _lib.load()
    assert lib.mdb_abi_struct_bytes(0) == C.sizeof(_lib.GemmDesc)
    assert lib.mdb_abi_struct_bytes(3) == C.sizeof(_lib.GemmBwdDesc)
    assert lib.mdb_abi_struct_bytes(8) == -1
    assert lib.mdb_abi_version() == 2


def test_im2col_kernels_do_not_spill_and_load_in_im2col_mode():
    from magicdance_b200 import build
    usage, bodies = _kernels(build.build())
    fwd = sorted(n for n in usage if "gemm_igemm_kernel" in n)
    bwd = sorted(n for n in usage if "gemm_bwd_igemm_kernel" in n)
    assert len(fwd) == 7 and len(bwd) == 2, (fwd, bwd)  # every tile width / ring depth the dispatch picks; dA, dB
    for name in fwd + bwd:
        assert usage[name] == (0, 0), f"{name}: LOCAL / STACK = {usage[name]}"
        assert "UTMALDG.4D.IM2COL" in bodies[name] and re.search(r"HGMMA\.64x\d+x16\.F32", bodies[name]), name
    for name in (n for n in usage if "gemm_tc_kernel" in n or re.search(r"gemm_bwd_kernelILi", n)):
        assert "IM2COL" not in bodies[name], f"{name}: the box-path kernels keep their tiled loads"


def _fwd(**over):
    """a 2 x 12 x 8 x 320 -> 320 conv descriptor whose pointers are never dereferenced"""
    from magicdance_b200 import _lib
    g = _lib.GemmDesc()
    g.a, g.b, g.d = 0x10000, 0x20000, 0x30000
    g.conv, g.nb, g.h, g.w, g.c = 1, 2, 12, 8, 320
    g.k1, g.ldb, g.ldd = 320, 2880, 320
    g.m, g.n, g.k = 2 * 12 * 8, 320, 2880
    for k, v in over.items():
        setattr(g, k, v)
    return g


FWD_REFUSALS = [
    (dict(conv=0), "conv must be the stride"),
    (dict(conv=3), "conv must be the stride"),
    (dict(c=100, k=900), "c % 64 == 0"),
    (dict(k=2816), "k == 9c"),
    (dict(m=100), "must be nb*ho*wo"),
    (dict(m=96, conv=2), "must be nb*ho*wo"),
    (dict(epilogue=1), "GEGLU"),
    (dict(ln_u=0x40000), "LayerNorm"),
    (dict(a2=0x40000, k1=100), "multiple of 64 below c"),
    (dict(a2=0x40000, k1=320), "multiple of 64 below c"),
    (dict(lda=100), "pixel strides"),
    (dict(a2=0x40000, k1=256, lda2=60), "pixel strides"),
    (dict(ldd=100), "ldd"),
    (dict(d=0x30004), "16B aligned"),
    (dict(bias=0x40004), "bias must be"),
    (dict(residual=0x40000, ldr=3), "residual must be"),
    (dict(b=0), "null operand"),
]


@pytest.mark.parametrize("over,msg", FWD_REFUSALS)
def test_forward_rejects_before_any_launch(over, msg):
    from magicdance_b200 import _lib
    lib = _lib.load()
    n0 = lib.mdb_launch_count()
    assert lib.mdb_conv3x3_igemm_f16(C.byref(_fwd(**over)), None) == -1
    assert msg.replace("%", "") in lib.mdb_last_error().decode().replace("%", "")
    assert lib.mdb_launch_count() == n0


def _bwd(**over):
    from magicdance_b200 import _lib
    g = _lib.GemmBwdDesc()
    f = g.fwd
    f.a, f.b = 0x10000, 0x20000
    f.conv, f.nb, f.h, f.w, f.c, f.k1, f.ldb = 1, 2, 12, 8, 320, 320, 2880
    f.m, f.n, f.k = 2 * 12 * 8, 320, 2880
    g.dd, g.lddd = 0x30000, 320
    g.da, g.ldda, g.db, g.lddb, g.db_dtype = 0x40000, 320, 0x50000, 2880, 1
    g.ws = 0x60000
    for k, v in over.items():
        setattr(f if k.startswith("fwd_") else g, k.removeprefix("fwd_"), v)
    return g


@pytest.mark.parametrize("over,msg", [
    (dict(fwd_conv=0), "conv must be the stride"),
    (dict(fwd_epilogue=1), "GEGLU"),
    (dict(fwd_k=2816), "k == 9c"),
    (dict(fwd_m=100), "m != nb"),
    (dict(fwd_a2=0x70000, fwd_k1=100), "multiple of 64 below c"),
    (dict(fwd_a2=0x70000, fwd_k1=256, fwd_conv=2, fwd_m=2 * 6 * 4), "stride-2 dA of a two-source conv"),
    (dict(da2=0x70000, ldda2=64), "da2 without a second source"),
    (dict(fwd_lda=12), "pixel strides"),
    (dict(lddd=100), "lddd"),
    (dict(db_dtype=2), "db must be"),
])
def test_backward_rejects_before_any_launch(over, msg):
    from magicdance_b200 import _lib
    lib = _lib.load()
    n0 = lib.mdb_launch_count()
    g = _bwd(**over)
    assert lib.mdb_conv3x3_igemm_bwd_f16(C.byref(g), None) == -1
    assert msg.replace("%", "") in lib.mdb_last_error().decode().replace("%", "")
    assert lib.mdb_conv3x3_igemm_bwd_ws_floats(C.byref(g)) == -1
    assert lib.mdb_launch_count() == n0


def test_backward_workspace_needs_no_column_buffer_at_stride_1():
    """12x8 takes dA and dB through im2col loads (no [M][9c] column buffer, unlike mdb_gemm_bwd_f16); stride-2 dA
    keeps the fp32 column buffer"""
    from magicdance_b200 import _lib
    lib = _lib.load()
    g = _bwd(splits=1, fwd_splits=1)
    assert lib.mdb_conv3x3_igemm_bwd_ws_floats(C.byref(g)) == 0
    assert lib.mdb_gemm_bwd_ws_floats(C.byref(g)) > 0
    g = _bwd(splits=1, fwd_splits=1, fwd_conv=2, fwd_m=2 * 6 * 4, db=None)
    assert lib.mdb_conv3x3_igemm_bwd_ws_floats(C.byref(g)) == 2 * 6 * 4 * 2880


def test_training_latent_sizes():
    from magicdance_b200.engine import NetConfig
    from magicdance_b200.train import check_latent_size
    for h, w in ((16, 16), (32, 32), (64, 64), (40, 24), (112, 64), (48, 48), (80, 80), (96, 96), (96, 64), (8, 8)):
        check_latent_size(NetConfig(), h, w)
    for h, w in ((12, 12), (100, 64), (64, 36), (0, 8)):
        with pytest.raises(ValueError, match="training forward"):
            check_latent_size(NetConfig(), h, w)


# ---------------------------------------------------------------------------------------------------------------------
# orchestration at 40x24 on the stand-ins
# ---------------------------------------------------------------------------------------------------------------------
def test_training_path_at_40x24_matches_the_reference_golden():
    """p_losses -> backward through train.py at 40x24, B = 2 (levels 40x24, 20x12, 10x6, 5x3: every tensor-core 3x3 conv
    on conv3x3_igemm_ad, the hint encoder's last conv included) against the UNMODIFIED reference's gradients
    (tests/golden/anysize40x24.npz, oracle/make_golden_anysize.py) at grad16's gates"""
    from magicdance_b200 import ops
    from tests import anysize_golden as A
    from tests import fake_igemm_ops, fake_train_ops
    from tests.test_train_cpu import TOL, stage2_model, train_step
    gold, inp = A.load()
    fake_igemm_ops.CALLS.clear()
    with pytest.MonkeyPatch.context() as mp:
        for name in fake_train_ops.PATCHED:
            mp.setattr(ops, name, getattr(fake_train_ops, name))
        mp.setattr(ops, "conv3x3_igemm_ad", fake_igemm_ops.conv3x3_igemm_ad)
        model = stage2_model()
        loss, _, dx, grads = train_step(model, {k: inp[k] for k in ("x0", "noise", "t_train", "context", "pose",
                                                                     "ref")})
        del model
    assert set(fake_igemm_ops.CALLS) == {(40, 24), (20, 12), (10, 6), (5, 3)}, fake_igemm_ops.CALLS
    A.compare_grads(gold, loss.detach(), dx, grads, TOL)


@pytest.fixture(scope="module")
def inference_model():
    """the stage-2 drop-in model with every kernel entry point of inference on the CPU stand-ins"""
    from magicdance_b200 import ops
    from tests import fake_igemm_ops, fake_ops
    from tests.test_engine_cpu import _PATCHED
    from tests.test_train_cpu import stage2_model

    def refuse(*a, **k):
        raise AssertionError("im2col3x3 called for a UNet conv")

    with pytest.MonkeyPatch.context() as mp, torch.no_grad():
        for name in _PATCHED + ("cfg_ddim_update",):
            mp.setattr(ops, name, getattr(fake_ops, name))
        mp.setattr(ops, "im2col3x3", refuse)
        mp.setattr(ops, "conv3x3_igemm", fake_igemm_ops.conv3x3_igemm)
        fake_igemm_ops.CALLS.clear()
        yield stage2_model().eval()


def test_apply_model_at_40x24_matches_the_reference_golden(inference_model):
    """apply_model (engine: bank, pose ControlNet, UNet) at 40x24, B = 2, per-sample t, with and without the reference
    latent, against the reference's eps"""
    from tests import anysize_golden as A
    from tests import fake_igemm_ops
    from tests import golden_util as G
    gold, inp = A.load()
    cond = {"c_concat": [inp["pose"]], "c_crossattn": [inp["context"]]}
    eps_c = inference_model.apply_model(inp["x"], inp["t"], cond, inp["ref"])
    eps_u = inference_model.apply_model(inp["x"], inp["t"], cond, None, uc=True)
    assert {(40, 24), (20, 12), (10, 6), (5, 3)} <= set(fake_igemm_ops.CALLS), fake_igemm_ops.CALLS
    e_c = G.rel_l2(eps_c, torch.from_numpy(gold["apply/eps_c"]))
    e_u = G.rel_l2(eps_u, torch.from_numpy(gold["apply/eps_u"]))
    print(f"40x24 eps rel-L2: cond {e_c:.3e}, uncond {e_u:.3e}")
    assert e_c <= 5e-3 and e_u <= 5e-3


def test_sampler_chain_at_40x24_matches_the_reference_golden(inference_model):
    """the drop-in DDIMSampler_ReferenceOnly.sample (what sample_log runs) for 4 DDIM steps at CFG 7 with a (4, 40, 24)
    shape, against the reference sampler's chain"""
    from magicdance_b200.dropin.ddim import DDIMSampler_ReferenceOnly
    from tests import anysize_golden as A
    from tests import golden_util as G
    gold, inp = A.load()
    c = {"c_concat": [inp["pose"][:1]], "c_crossattn": [inp["context"][:1]], "image_control": [inp["ref"][:1]],
         "wonoise": True, "overlap_sampling": False}
    uc = {"c_concat": [inp["pose"][:1]], "c_crossattn": [inp["uc_context"]], "wonoise": True, "overlap_sampling": False}
    try:
        x, inter = DDIMSampler_ReferenceOnly(inference_model).sample(
            4, 1, (4, 40, 24), c, verbose=False, eta=0.0, x_T=inp["x"][:1], unconditional_guidance_scale=7.0,
            unconditional_conditioning=uc)
    finally:
        inference_model.__dict__.pop("_mdb_pipelines", None)
    e_x = G.rel_l2(x, torch.from_numpy(gold["chain/x"]))
    e_p = G.rel_l2(inter["pred_x0"][-1], torch.from_numpy(gold["chain/pred_x0"]))
    print(f"40x24 4-step chain rel-L2: x {e_x:.3e}, pred_x0 {e_p:.3e}")
    assert e_x <= 1e-2 and e_p <= 1e-2
