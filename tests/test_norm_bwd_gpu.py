"""GroupNorm / LayerNorm / GEGLU backward on the GPU: per-shape gradient numerics (tests/norm_bwd_cases.py),
bit-reproducibility, and two blocks differentiated end to end through library kernels against the fp32 restatement
(oracle/restatement.py): an output-block ResBlock and a read-mode SpatialTransformer."""
import pytest
import torch
import torch.nn.functional as F

from oracle import restatement as R
from tests import norm_bwd_cases as N
from tests.kernel_cases import _rand, rel

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", N.CASES, ids=[N.case_id(c) for c in N.CASES])
def test_backward_matches_torch_fp64(case):
    fn, kw = case
    err, tol, desc = fn(**kw)
    torch.cuda.synchronize()
    print(desc)
    assert err <= tol, f"{desc}: error {err:.3e} > {tol:.1e}"


def test_backward_is_bit_reproducible():
    """every output of a repeated call is bit-equal (fixed-order reductions, no atomics)"""
    from magicdance_b200 import ops
    b, hw, c1, c2 = 4, 1024, 640, 320
    x1, x2 = _rand(b * hw, c1, seed=1).half(), _rand(b * hw, c2, seed=2).half()
    gamma, beta = _rand(c1 + c2, seed=3).float(), _rand(c1 + c2, seed=4).float()
    dy = _rand(b * hw, c1 + c2, seed=5).half()
    kw = dict(batch=b, hw=hw, eps=1e-5, silu=True, x2=x2)
    x, g, dyl = _rand(4096, 1280, seed=6).half(), _rand(1280, seed=7).float(), _rand(4096, 1280, seed=8).half()
    h, dout = _rand(1000, 2560, seed=9).half(), _rand(1000, 1280, seed=10).half()
    runs = [ops.groupnorm_backward(x1, gamma, beta, dy, **kw) + ops.layernorm_backward(x, g, dyl) +
            (ops.geglu(h), ops.geglu_backward(h, dout)) for _ in range(2)]
    torch.cuda.synchronize()
    for a, b_ in zip(*runs):
        assert torch.equal(a, b_)


def _params(spec, seed):
    """{name: fp32 tensor on the GPU, rounded through fp16} for (name, shape, scale) — scale None: 1 + 0.2 N(0, 1)
    (norm weights)"""
    sd = {}
    for i, (nm, shape, scale) in enumerate(spec):
        t = 1 + 0.2 * _rand(*shape, seed=seed + i) if scale is None else _rand(*shape, seed=seed + i, scale=scale)
        sd[nm] = t.half().float()
    return sd


def _leaves(sd):
    return {k: v.clone().requires_grad_() for k, v in sd.items()}


def _nhwc(t):
    """NCHW -> [B*H*W, C]"""
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def _check(errs):
    print({k: f"{v:.2e}" for k, v in errs.items()})
    assert max(errs.values()) <= 1e-2, errs


def test_output_block_resblock_backward():
    """[h | skip] -> group_norm+SiLU (dual source) -> 3x3 conv with the per-sample emb bias -> group_norm+SiLU ->
    3x3 conv + the 1x1 skip conv of the concat: dh, dskip and every parameter gradient against R.resblock in fp32"""
    with torch.enable_grad():  # other tests switch autograd off process-wide
        _resblock()


def _resblock():
    from magicdance_b200 import ops
    b, hh, ww, ch, cs, co, ce = 2, 16, 16, 320, 320, 320, 128
    ci, hw = ch + cs, hh * ww
    sd = _params([("in_layers.0.weight", (ci,), None), ("in_layers.0.bias", (ci,), 0.2),
                  ("in_layers.2.weight", (co, ci, 3, 3), (9 * ci) ** -0.5), ("in_layers.2.bias", (co,), 0.1),
                  ("emb_layers.1.weight", (co, ce), ce ** -0.5), ("emb_layers.1.bias", (co,), 0.1),
                  ("out_layers.0.weight", (co,), None), ("out_layers.0.bias", (co,), 0.2),
                  ("out_layers.3.weight", (co, co, 3, 3), (9 * co) ** -0.5), ("out_layers.3.bias", (co,), 0.1),
                  ("skip_connection.weight", (co, ci, 1, 1), ci ** -0.5), ("skip_connection.bias", (co,), 0.1)],
                 seed=10)
    h = _rand(b * hw, ch, seed=1).half()
    skip = _rand(b * hw, cs, seed=2).half()
    emb = _rand(b, ce, seed=3)
    g = _rand(b * hw, co, seed=4)

    p = _leaves(sd)
    xs = [t.clone().requires_grad_() for t in (h, skip)]
    a = ops.group_norm(xs[0], p["in_layers.0.weight"], p["in_layers.0.bias"], batch=b, hw=hw, eps=1e-5, silu=True,
                       x2=xs[1])
    e = F.linear(F.silu(emb), p["emb_layers.1.weight"], p["emb_layers.1.bias"]) + p["in_layers.2.bias"]
    a = ops.tc_gemm(a, ops.pack_conv_weight(p["in_layers.2.weight"]), w_param=p["in_layers.2.weight"], bias=e.contiguous(),
                    bias_batch_stride=co, rows_per_batch=hw, conv=(b, hh, ww, ci))
    a = ops.group_norm(a, p["out_layers.0.weight"], p["out_layers.0.bias"], batch=b, hw=hw, eps=1e-5, silu=True)
    wsk = p["skip_connection.weight"]
    res = ops.tc_gemm(xs[0], wsk.detach().view(co, ci).half(), w_param=wsk.view(co, ci), a2=xs[1],
                      bias=p["skip_connection.bias"])
    out = ops.tc_gemm(a, ops.pack_conv_weight(p["out_layers.3.weight"]), w_param=p["out_layers.3.weight"],
                      bias=p["out_layers.3.bias"], residual=res, conv=(b, hh, ww, co))
    (out.float() * g).sum().backward()

    r = _leaves(sd)
    rh, rs = (t.float().view(b, hh, ww, -1).permute(0, 3, 1, 2).contiguous().requires_grad_() for t in (h, skip))
    ref = R.resblock(r, "", torch.cat([rh, rs], 1), emb)
    (_nhwc(ref) * g).sum().backward()
    errs = {"dh": rel(xs[0].grad.float(), _nhwc(rh.grad)), "dskip": rel(xs[1].grad.float(), _nhwc(rs.grad))}
    for k in sd:
        assert p[k].grad.shape == r[k].grad.shape and p[k].grad.dtype == torch.float32, k
        errs[k] = rel(p[k].grad, r[k].grad)
    _check(errs)


def test_read_mode_spatial_transformer_backward():
    """GroupNorm (eps 1e-6) -> proj_in -> LN1 -> q / k / V^T -> two-source attention over [self | bank] -> to_out ->
    LN2 -> to_q (unfolded) -> attention over the per-sample context -> to_out -> LN3 -> GEGLU proj -> geglu -> ff out
    -> proj_out + x: dx, dbank, dcontext and every parameter gradient against R.spatial_transformer in fp32"""
    with torch.enable_grad():
        _spatial_transformer()


def _spatial_transformer():
    from magicdance_b200 import ops
    b, hh, ww, c, heads, nb, nt, cd = 2, 16, 16, 320, 8, 256, 80, 64
    d, n, ff = c // heads, hh * ww, 4 * c
    tb = "transformer_blocks.0."
    spec = [("norm.weight", (c,), None), ("norm.bias", (c,), 0.2),
            ("proj_in.weight", (c, c, 1, 1), c ** -0.5), ("proj_in.bias", (c,), 0.1),
            ("proj_out.weight", (c, c, 1, 1), c ** -0.5), ("proj_out.bias", (c,), 0.1)]
    for i in (1, 2, 3):
        spec += [(f"{tb}norm{i}.weight", (c,), None), (f"{tb}norm{i}.bias", (c,), 0.2)]
    for at, kd in (("attn1", c), ("attn2", cd)):
        spec += [(f"{tb}{at}.to_q.weight", (c, c), c ** -0.5), (f"{tb}{at}.to_k.weight", (c, kd), kd ** -0.5),
                 (f"{tb}{at}.to_v.weight", (c, kd), kd ** -0.5), (f"{tb}{at}.to_out.0.weight", (c, c), c ** -0.5),
                 (f"{tb}{at}.to_out.0.bias", (c,), 0.1)]
    spec += [(f"{tb}ff.net.0.proj.weight", (2 * ff, c), c ** -0.5), (f"{tb}ff.net.0.proj.bias", (2 * ff,), 0.1),
             (f"{tb}ff.net.2.weight", (c, ff), ff ** -0.5), (f"{tb}ff.net.2.bias", (c,), 0.1)]
    sd = _params(spec, seed=20)
    x = _rand(b * n, c, seed=1).half()
    bank = _rand(b * nb, c, seed=2).half()
    ctx = _rand(b * nt, cd, seed=3).half()
    g = _rand(b * n, c, seed=4)

    p = _leaves(sd)
    xs = [t.clone().requires_grad_() for t in (x, bank, ctx)]
    lin = lambda a, nm, **kw: ops.tc_gemm(a, p[nm].detach().reshape(p[nm].shape[0], -1).half(),
                                          w_param=p[nm].view(p[nm].shape[0], -1), **kw)
    vt = lambda nm, a: ops.tc_gemm(p[nm].detach().half(), a, a_param=p[nm])  # V^T = W_v a^T
    ln = lambda a, i: ops.layer_norm(a, p[f"{tb}norm{i}.weight"], p[f"{tb}norm{i}.bias"])
    akw = dict(heads=heads, d=d, batch=b, nq=n)

    y = ops.group_norm(xs[0], p["norm.weight"], p["norm.bias"], batch=b, hw=n, eps=1e-6, silu=False)
    y = lin(y, "proj_in.weight", bias=p["proj_in.bias"])
    n1 = ln(y, 1)
    a1 = f"{tb}attn1."
    o = ops.two_source_attention(lin(n1, a1 + "to_q.weight"), lin(n1, a1 + "to_k.weight"), vt(a1 + "to_v.weight", n1),
                                 n, k1=lin(xs[1], a1 + "to_k.weight"), vt1=vt(a1 + "to_v.weight", xs[1]), n1=nb,
                                 kv1_batches=b, bank_batches=b, **akw)
    y = lin(o, a1 + "to_out.0.weight", bias=p[a1 + "to_out.0.bias"], residual=y)
    a2 = f"{tb}attn2."
    o = ops.two_source_attention(lin(ln(y, 2), a2 + "to_q.weight"), lin(xs[2], a2 + "to_k.weight"),
                                 vt(a2 + "to_v.weight", xs[2]), nt, **akw)
    y = lin(o, a2 + "to_out.0.weight", bias=p[a2 + "to_out.0.bias"], residual=y)
    hproj = lin(ln(y, 3), f"{tb}ff.net.0.proj.weight", bias=p[f"{tb}ff.net.0.proj.bias"])
    y = lin(ops.geglu(hproj), f"{tb}ff.net.2.weight", bias=p[f"{tb}ff.net.2.bias"], residual=y)
    out = lin(y, "proj_out.weight", bias=p["proj_out.bias"], residual=xs[0])
    (out.float() * g).sum().backward()

    r = _leaves(sd)
    rx = x.float().view(b, hh, ww, c).permute(0, 3, 1, 2).contiguous().requires_grad_()
    rb = bank.float().view(b, nb, c).requires_grad_()
    rc = ctx.float().view(b, nt, cd).requires_grad_()
    ref = R.spatial_transformer(r, "", rx, rc, heads, "read", None, [rb])
    (_nhwc(ref) * g).sum().backward()
    errs = {"dx": rel(xs[0].grad.float(), _nhwc(rx.grad)), "dbank": rel(xs[1].grad.float(), rb.grad),
            "dcontext": rel(xs[2].grad.float(), rc.grad)}
    for k in sd:
        assert p[k].grad.shape == r[k].grad.shape and p[k].grad.dtype == torch.float32, k
        errs[k] = rel(p[k].grad, r[k].grad)
    _check(errs)


def test_groupnorm_backward_calls_of_different_shapes_share_one_workspace():
    """the statistics kernel's tickets reset themselves: a big, a small and again the big call on one "gn_bwd"
    workspace give the bits of the same calls on fresh, zeroed workspaces (their own scratch lanes)"""
    from magicdance_b200 import ops
    shapes = [dict(batch=4, hw=1024, c1=640, c2=320), dict(batch=1, hw=15, c1=2560),
              dict(batch=4, hw=1024, c1=640, c2=320)]

    def call(batch, hw, c1, c2=0, seed=0):
        x1 = _rand(batch * hw, c1, seed=seed).half()
        x2 = _rand(batch * hw, c2, seed=seed + 1).half() if c2 else None
        g, b = _rand(c1 + c2, seed=seed + 2).float(), _rand(c1 + c2, seed=seed + 3).float()
        dy = _rand(batch * hw, c1 + c2, seed=seed + 4).half()
        return ops.groupnorm_backward(x1, g, b, dy, batch=batch, hw=hw, eps=1e-5, silu=True, x2=x2)

    shared = [call(**s, seed=i) for i, s in enumerate(shapes)]
    fresh = []
    for i, s in enumerate(shapes):
        with ops.workspace_lane(("gn_bwd_fresh", i)):
            fresh.append(call(**s, seed=i))
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(shared, fresh)):
        for x, y in zip(a, b):
            assert (x is None and y is None) or torch.equal(x, y), f"call {i} ({shapes[i]})"
