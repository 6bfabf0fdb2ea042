"""Numerics cases of the GroupNorm(+SiLU) / LayerNorm / GEGLU backward (ops.groupnorm_backward, ops.layernorm_backward,
ops.geglu / ops.geglu_backward): each case runs the library on the GPU and returns (error, tolerance, description)
against torch float64 autograd of F.group_norm / F.silu, F.layer_norm, or chunk + F.gelu computed from the SAME
fp16-rounded inputs.  Run by tests/test_norm_bwd_gpu.py; the same (error, tolerance, description) contract as
tests/kernel_cases.py.  The error is the largest rel-L2 over the outputs; fp16 outputs are gated at the forward
kernels' 2e-3, fp32 outputs (dx in fp32, dgamma, dbeta) at 5e-4."""
import torch
import torch.nn.functional as F

from magicdance_b200 import ops
from tests.kernel_cases import DEV, _rand, rel

TOL = 2e-3
TOL_F32 = 5e-4
_DT = {"f16": torch.float16, "f32": torch.float32}


def _errs_desc(errs):
    return " ".join(f"{nm} {e:.2e}" for nm, e in errs.items())


def _gate(errs, tols, desc):
    """(error of the output closest to its gate, that gate, description)"""
    worst = max(errs, key=lambda k: errs[k] / tols[k])
    return errs[worst], tols[worst], f"{desc}: rel-L2 {_errs_desc(errs)}"


def case_gn_bwd(batch, hw, c1, c2=0, eps=1e-5, silu=True, mean=0.0, spread=1.0, dx_dtype="f16", accumulate=(),
                seed=0):
    """GroupNorm(32) [+SiLU] backward over [x1 | x2]; mean / spread shape the activations (mean 40, spread 1.5 is the
    cancellation case the forward's pivot shift exists for); accumulate: gradients added into random destinations"""
    c = c1 + c2
    x1 = (_rand(batch * hw, c1, seed=seed) * spread + mean).half()
    x2 = (_rand(batch * hw, c2, seed=seed + 1) * spread + mean).half() if c2 else None
    gamma = (1 + 0.2 * _rand(c, seed=seed + 2)).float()
    beta = (0.2 * _rand(c, seed=seed + 3)).float()
    dy = _rand(batch * hw, c, seed=seed + 4).half()
    kw = dict(batch=batch, hw=hw, eps=eps, silu=silu, x2=x2, dx_dtype=_DT[dx_dtype], accumulate=accumulate)
    init = {}
    shapes = {"x": (batch * hw, c1), "x2": (batch * hw, c2), "gamma": (c,), "beta": (c,)}
    for i, nm in enumerate(accumulate):
        dt = torch.float32 if nm in ("gamma", "beta") else _DT[dx_dtype]
        init[nm] = _rand(*shapes[nm], seed=seed + 5 + i).to(dt)
        kw[{"x": "out_dx1", "x2": "out_dx2", "gamma": "out_dgamma", "beta": "out_dbeta"}[nm]] = init[nm].clone()
    dx1, dx2, dgamma, dbeta = ops.groupnorm_backward(x1, gamma, beta, dy, **kw)

    with torch.enable_grad():  # other tests switch autograd off process-wide
        xs = [x1.double().requires_grad_()] + ([x2.double().requires_grad_()] if c2 else [])
        g64, b64 = gamma.double().requires_grad_(), beta.double().requires_grad_()
        x = torch.cat(xs, 1).view(batch, hw, c).permute(0, 2, 1)
        y = F.group_norm(x, 32, g64, b64, eps)
        if silu:
            y = F.silu(y)
        (y.permute(0, 2, 1).reshape(batch * hw, c) * dy.double()).sum().backward()
    refs = {"x": xs[0].grad, "gamma": g64.grad, "beta": b64.grad}
    if c2:
        refs["x2"] = xs[1].grad
    got = {"x": dx1, "x2": dx2, "gamma": dgamma, "beta": dbeta}
    errs, tols = {}, {}
    for nm, ref in refs.items():
        base = init.get(nm)
        errs["d" + nm] = rel(got[nm].double(), ref if base is None else base.double() + ref)
        tols["d" + nm] = TOL if got[nm].dtype == torch.float16 else TOL_F32
    desc = (f"groupnorm backward B={batch} hw={hw} c={c1}+{c2} eps={eps} silu={silu} mean={mean} spread={spread} "
            f"dx={dx_dtype} acc={','.join(accumulate)}")
    return _gate(errs, tols, desc)


def case_ln_bwd(rows, c, mean=0.0, spread=1.0, dx_dtype="f16", accumulate=(), seed=0):
    x = (_rand(rows, c, seed=seed) * spread + mean).half()
    gamma = (1 + 0.2 * _rand(c, seed=seed + 1)).float()
    beta = (0.2 * _rand(c, seed=seed + 2)).float()
    dy = _rand(rows, c, seed=seed + 3).half()
    kw = dict(dx_dtype=_DT[dx_dtype], accumulate=accumulate)
    init = {}
    for i, nm in enumerate(accumulate):
        dt = torch.float32 if nm in ("gamma", "beta") else _DT[dx_dtype]
        init[nm] = _rand(*((rows, c) if nm == "x" else (c,)), seed=seed + 4 + i).to(dt)
        kw["out_d" + nm] = init[nm].clone()
    dx, dgamma, dbeta = ops.layernorm_backward(x, gamma, dy, **kw)

    with torch.enable_grad():
        x64, g64, b64 = (t.double().requires_grad_() for t in (x, gamma, beta))
        (F.layer_norm(x64, (c,), g64, b64, 1e-5) * dy.double()).sum().backward()
    errs, tols = {}, {}
    for nm, got, ref in (("x", dx, x64.grad), ("gamma", dgamma, g64.grad), ("beta", dbeta, b64.grad)):
        base = init.get(nm)
        errs["d" + nm] = rel(got.double(), ref if base is None else base.double() + ref)
        tols["d" + nm] = TOL if got.dtype == torch.float16 else TOL_F32
    desc = f"layernorm backward rows={rows} c={c} mean={mean} spread={spread} dx={dx_dtype} acc={','.join(accumulate)}"
    return _gate(errs, tols, desc)


def case_geglu(m, n, seed=0):
    """forward out = v * gelu(g) and backward dh = [dv | dg] of h = [v | g] in the projection's row order"""
    h = _rand(m, 2 * n, seed=seed).half()
    dout = _rand(m, n, seed=seed + 1).half()
    out = ops.geglu(h)
    dh = ops.geglu_backward(h, dout)
    with torch.enable_grad():
        h64 = h.double().requires_grad_()
        v, g = h64.chunk(2, dim=-1)
        ref = v * F.gelu(g)
        (ref * dout.double()).sum().backward()
    errs = {"out": rel(out.double(), ref.detach()), "dh": rel(dh.double(), h64.grad)}
    return _gate(errs, {"out": TOL, "dh": TOL}, f"geglu m={m} n={n}")


# (case function, keyword arguments); config-5 sizes are batch 4 at a 64x64 latent
CASES = [
    # every GroupNorm width at batch 4 and its training HW (64x64 / 32x32 / 16x16 / 8x8 levels)
    (case_gn_bwd, dict(batch=4, hw=4096, c1=320)),
    (case_gn_bwd, dict(batch=4, hw=1024, c1=640)),
    (case_gn_bwd, dict(batch=4, hw=4096, c1=960)),
    (case_gn_bwd, dict(batch=4, hw=256, c1=1280)),
    (case_gn_bwd, dict(batch=4, hw=1024, c1=1920)),
    (case_gn_bwd, dict(batch=4, hw=64, c1=2560)),
    # the output blocks' fused [h | skip] concat
    (case_gn_bwd, dict(batch=4, hw=4096, c1=320, c2=320)),
    (case_gn_bwd, dict(batch=4, hw=4096, c1=640, c2=320)),
    (case_gn_bwd, dict(batch=4, hw=1024, c1=1280, c2=640)),
    (case_gn_bwd, dict(batch=4, hw=256, c1=1280, c2=1280)),
    # SpatialTransformer's Normalize: eps 1e-6, no SiLU
    (case_gn_bwd, dict(batch=4, hw=4096, c1=320, eps=1e-6, silu=False)),
    # ragged HW, and stage 1's batch of 32
    (case_gn_bwd, dict(batch=3, hw=1000, c1=640)),
    (case_gn_bwd, dict(batch=32, hw=256, c1=1280)),
    # large mean against the spread
    (case_gn_bwd, dict(batch=4, hw=1024, c1=640, mean=40.0, spread=1.5)),
    (case_gn_bwd, dict(batch=2, hw=256, c1=640, c2=640, mean=40.0, spread=1.5, silu=False, eps=1e-6)),
    # fp32 and accumulating destinations
    (case_gn_bwd, dict(batch=2, hw=1024, c1=640, c2=320, dx_dtype="f32", accumulate=("x", "x2", "gamma", "beta"))),
    (case_gn_bwd, dict(batch=2, hw=256, c1=1280, accumulate=("x",))),
    (case_gn_bwd, dict(batch=2, hw=256, c1=1280, dx_dtype="f32")),
]
for _c in (320, 640, 1280):
    CASES += [(case_ln_bwd, dict(rows=r, c=_c)) for r in (16384, 4096, 1024, 256, 1000)]
CASES += [
    (case_ln_bwd, dict(rows=4096, c=320, mean=40.0, spread=1.5)),
    (case_ln_bwd, dict(rows=1024, c=1280, mean=40.0, spread=1.5)),
    (case_ln_bwd, dict(rows=1024, c=640, dx_dtype="f32", accumulate=("x", "gamma", "beta"))),
    (case_ln_bwd, dict(rows=1000, c=320, accumulate=("x",))),
    # GEGLU: (tokens, N) of the three levels' FF (N = 4 C) at batch 4, and a ragged M
    (case_geglu, dict(m=16384, n=1280)),
    (case_geglu, dict(m=4096, n=2560)),
    (case_geglu, dict(m=1024, n=5120)),
    (case_geglu, dict(m=1000, n=1280)),
]


def case_id(case):
    fn, kw = case
    return fn.__name__.removeprefix("case_") + "-" + "-".join(f"{k}={v}" for k, v in kw.items()).replace(
        " ", "").replace("'", "")
