"""Numerics cases of the GroupNorm(+SiLU) / LayerNorm / GEGLU backward (ops.groupnorm_backward, ops.layernorm_backward,
ops.geglu / ops.geglu_backward): each case runs the library on the GPU and returns (error, tolerance, description)
against torch float64 autograd of F.group_norm / F.silu, F.layer_norm, or chunk + F.gelu computed from the SAME
fp16-rounded inputs.  Run by tests/test_norm_bwd_gpu.py; the same (error, tolerance, description) contract as
tests/kernel_cases.py.  The error is the largest rel-L2 over the outputs; fp16 outputs are gated at the forward
kernels' 2e-3, fp32 outputs (dx in fp32, dgamma, dbeta) at 5e-4.

Every output goes into a NaN-poisoned, guarded buffer or a poisoned allocation (tests/kernel_guard.py), so an element
that is never written, or a write outside the output, fails the case.  dx is gated per block as well: per (sample,
group) for GroupNorm, per 128 rows x 32 channels for LayerNorm; GEGLU's strided h and dout hold NaN in their
row-stride padding; the LayerNorm workspace holds NaN before each call (the GroupNorm one must start at zero); every
call runs twice and must be bit-equal."""
import torch
import torch.nn.functional as F

from magicdance_b200 import ops
from tests.kernel_cases import DEV, _rand, nan_padded
from tests.kernel_guard import (Guarded, bit_equal, check_poisoned, check_workspace_used, gated, poison_workspace,
                                poisoned_alloc, rel)

TOL = 2e-3
TOL_F32 = 5e-4
_DT = {"f16": torch.float16, "f32": torch.float32}


def _errs_desc(errs):
    return " ".join(f"{nm} {e:.2e}" for nm, e in errs.items())


def _gate(errs, tols, desc):
    """(error of the output closest to its gate, that gate, description)"""
    worst = max(errs, key=lambda k: errs[k] / tols[k])
    return errs[worst], tols[worst], f"{desc}: error {_errs_desc(errs)}"


def _twice(launch, specs, init, desc):
    """launch(outs) twice, each time into fresh Guarded destinations (specs: {name: (rows, cols, dtype, shape)},
    contiguous; names in init start from those contents); both runs must be bit-equal.  Returns {name: output}."""
    runs = []
    for what in ("", " (second run)"):
        g = {nm: Guarded(r, c, dt, contiguous=True, shape=shape) for nm, (r, c, dt, shape) in specs.items()}
        for nm, t in init.items():
            g[nm].out.copy_(t)
        launch({nm: t.out for nm, t in g.items()})
        for nm, t in g.items():
            t.check(f"{desc} d{nm}{what}")
        runs.append({nm: t.out for nm, t in g.items()})
    for nm in specs:
        if not bit_equal(runs[0][nm], runs[1][nm]):
            raise AssertionError(f"{desc}: d{nm} differs between two runs")
    return runs[0]


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
    specs = {"x": (batch * hw, c1, _DT[dx_dtype], None), "gamma": (1, c, torch.float32, (c,)),
             "beta": (1, c, torch.float32, (c,))}
    if c2:
        specs["x2"] = (batch * hw, c2, _DT[dx_dtype], None)
    init = {}
    for i, nm in enumerate(accumulate):
        r, cc, dt, shape = specs[nm]
        init[nm] = _rand(*(shape or (r, cc)), seed=seed + 5 + i).to(dt)
    desc = (f"groupnorm backward B={batch} hw={hw} c={c1}+{c2} eps={eps} silu={silu} mean={mean} spread={spread} "
            f"dx={dx_dtype} acc={','.join(accumulate)}")
    out_kw = {"x": "out_dx1", "x2": "out_dx2", "gamma": "out_dgamma", "beta": "out_dbeta"}
    got = _twice(lambda o: ops.groupnorm_backward(x1, gamma, beta, dy, **kw, **{out_kw[k]: v for k, v in o.items()}),
                 specs, init, desc)

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
    refs = {nm: ref if nm not in init else init[nm].double() + ref for nm, ref in refs.items()}
    errs, tols = {}, {}
    for nm, ref in refs.items():
        errs["d" + nm] = rel(got[nm].double(), ref)
        tols["d" + nm] = TOL if got[nm].dtype == torch.float16 else TOL_F32
    # [dx1 | dx2] per (sample, group): the groups of the concat straddle the x1 / x2 boundary
    dx = torch.cat([got["x"]] + ([got["x2"]] if c2 else []), 1).double()
    rx = torch.cat([refs["x"]] + ([refs["x2"]] if c2 else []), 1)
    e, note = gated(dx, rx, tols["dx"], rows=hw, cols=c // 32, groups=batch)
    errs["dx(gated)"], tols["dx(gated)"] = e, tols["dx"]
    return _gate(errs, tols, desc + note)


def case_ln_bwd(rows, c, mean=0.0, spread=1.0, dx_dtype="f16", accumulate=(), seed=0):
    x = (_rand(rows, c, seed=seed) * spread + mean).half()
    gamma = (1 + 0.2 * _rand(c, seed=seed + 1)).float()
    beta = (0.2 * _rand(c, seed=seed + 2)).float()
    dy = _rand(rows, c, seed=seed + 3).half()
    kw = dict(dx_dtype=_DT[dx_dtype], accumulate=accumulate)
    specs = {"x": (rows, c, _DT[dx_dtype], None), "gamma": (1, c, torch.float32, (c,)),
             "beta": (1, c, torch.float32, (c,))}
    init = {}
    for i, nm in enumerate(accumulate):
        r, cc, dt, shape = specs[nm]
        init[nm] = _rand(*(shape or (r, cc)), seed=seed + 4 + i).to(dt)
    desc = f"layernorm backward rows={rows} c={c} mean={mean} spread={spread} dx={dx_dtype} acc={','.join(accumulate)}"

    def launch(o):
        ws = poison_workspace("ln_bwd", device=x.device)
        ops.layernorm_backward(x, gamma, dy, **kw, **{"out_d" + k: v for k, v in o.items()})
        launch.ws = ws
    got = _twice(launch, specs, init, desc)
    check_workspace_used("ln_bwd", launch.ws, desc, x.device)

    with torch.enable_grad():
        x64, g64, b64 = (t.double().requires_grad_() for t in (x, gamma, beta))
        (F.layer_norm(x64, (c,), g64, b64, 1e-5) * dy.double()).sum().backward()
    errs, tols, note = {}, {}, ""
    for nm, ref in (("x", x64.grad), ("gamma", g64.grad), ("beta", b64.grad)):
        base = init.get(nm)
        ref = ref if base is None else base.double() + ref
        tols["d" + nm] = TOL if got[nm].dtype == torch.float16 else TOL_F32
        if nm == "x":
            errs["dx"], note = gated(got[nm].double(), ref, tols["dx"])
        else:
            errs["d" + nm] = rel(got[nm].double(), ref)
    return _gate(errs, tols, desc + note)


def case_geglu(m, n, seed=0):
    """forward out = v * gelu(g) and backward dh = [dv | dg] of h = [v | g] in the projection's row order; h and dout
    are column slices of wider NaN-padded buffers, and out and dh land in poisoned allocations"""
    h = nan_padded(_rand(m, 2 * n, seed=seed).half())
    dout = nan_padded(_rand(m, n, seed=seed + 1).half())
    desc = f"geglu m={m} n={n}"
    runs = []
    for what in ("", " (second run)"):
        ptr = poisoned_alloc((m, n), torch.float16)
        out = ops.geglu(h)
        check_poisoned(out, ptr, desc + " out" + what)
        ptr = poisoned_alloc((m, 2 * n), torch.float16)
        dh = ops.geglu_backward(h, dout)
        check_poisoned(dh, ptr, desc + " dh" + what)
        runs.append((out, dh))
    for nm, a, b in zip(("out", "dh"), *runs):
        if not bit_equal(a, b):
            raise AssertionError(f"{desc}: {nm} differs between two runs")
    out, dh = runs[0]
    with torch.enable_grad():
        h64 = h.double().requires_grad_()
        v, g = h64.chunk(2, dim=-1)
        ref = v * F.gelu(g)
        (ref * dout.double()).sum().backward()
    e_out, n_out = gated(out.double(), ref.detach(), TOL)
    e_dh, n_dh = gated(dh.double(), h64.grad, TOL)
    return _gate({"out": e_out, "dh": e_dh}, {"out": TOL, "dh": TOL}, f"{desc}: out{n_out} dh{n_dh}")


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
CASES += [
    # the GroupNorm token counts of a 40x24 latent (960 / 240 / 60 / 15 per level), single and dual source, up to the
    # widest group (c = 2560), and batch 1
    (case_gn_bwd, dict(batch=2, hw=960, c1=320)),
    (case_gn_bwd, dict(batch=2, hw=960, c1=320, c2=320)),
    (case_gn_bwd, dict(batch=2, hw=960, c1=640, c2=320)),
    (case_gn_bwd, dict(batch=2, hw=240, c1=640)),
    (case_gn_bwd, dict(batch=2, hw=240, c1=1280, c2=640)),
    (case_gn_bwd, dict(batch=2, hw=60, c1=1280)),
    (case_gn_bwd, dict(batch=2, hw=60, c1=1280, c2=1280)),
    (case_gn_bwd, dict(batch=2, hw=15, c1=2560)),
    (case_gn_bwd, dict(batch=2, hw=15, c1=1280, c2=1280, eps=1e-6, silu=False)),
    (case_gn_bwd, dict(batch=1, hw=15, c1=1280, c2=640)),
    (case_gn_bwd, dict(batch=1, hw=4096, c1=320)),
    (case_gn_bwd, dict(batch=1, hw=60, c1=2560, dx_dtype="f32")),
]
# LayerNorm over 1, 7, 15 and 30 rows (30: a 40x24 latent's deepest level at batch 2)
CASES += [(case_ln_bwd, dict(rows=_r, c=_c)) for _c in (320, 640, 1280) for _r in (1, 7, 15, 30)]
# GEGLU over 1, 7 and 77 rows
CASES += [(case_geglu, dict(m=_m, n=1280)) for _m in (1, 7, 77)]


def case_id(case):
    fn, kw = case
    return fn.__name__.removeprefix("case_") + "-" + "-".join(f"{k}={v}" for k, v in kw.items()).replace(
        " ", "").replace("'", "")
