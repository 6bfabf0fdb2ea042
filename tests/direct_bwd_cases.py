"""Numerics cases of the direct-conv, skinny-Linear and upsample backward (ops.conv3x3_direct_backward,
ops.direct_conv3x3, ops.skinny_linear_backward, ops.upsample2x_backward): each case runs the library on the GPU and
returns (error, tolerance, description) against torch float64 autograd of F.conv2d / F.silu, F.linear or
F.interpolate(nearest) computed from the SAME fp16-rounded inputs.  Run by tests/test_direct_bwd_gpu.py.  Every output
goes into a NaN-poisoned, guarded buffer (tests/kernel_guard.py), so an element that is never written, or a write
outside the output, fails the case.  fp16 outputs are gated at 3e-3 rel-L2, fp32 outputs (dW, dbias, the skinny
gradients, fp32 upsample dx) at 2e-3."""
import torch
import torch.nn.functional as F

from magicdance_b200 import ops
from tests.kernel_cases import _rand
from tests.kernel_guard import Guarded, gated, rel

TOL = 3e-3
TOL_F32 = 2e-3

# the ControlNet hint encoder's direct convs (cldm.py:599-615) as (cin, cout, stride, input size / pose-map size); a
# SiLU follows each; the eighth conv, 256 -> 320, runs on the tensor-core GEMM
HINT_LAYERS = [(3, 16, 1, 1), (16, 16, 1, 1), (16, 32, 2, 1), (32, 32, 1, 2), (32, 96, 2, 2), (96, 96, 1, 4),
               (96, 256, 2, 4)]


def _gate(errs, tols, desc):
    worst = max(errs, key=lambda k: errs[k] / tols[k])
    return errs[worst], tols[worst], f"{desc}: rel-L2 " + " ".join(f"{k} {v:.2e}" for k, v in errs.items())


def _conv_inputs(batch, h, w, cin, cout, stride, bias, seed):
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    x = _rand(batch * h * w, cin, seed=seed).half()
    wp = _rand(cout, cin, 3, 3, seed=seed + 1, scale=(9 * cin) ** -0.5).half().float()  # OIHW, fp16-rounded
    wt = wp.permute(0, 2, 3, 1).reshape(cout, 9 * cin).half().contiguous()
    b = _rand(cout, seed=seed + 2, scale=0.3).float() if bias else None
    dy = _rand(batch * ho * wo, cout, seed=seed + 3).half()
    return x, wp, wt, b, dy, ho, wo


def _conv_ref(x, wp, b, dy, batch, h, w, cin, cout, stride, silu, ho, wo):
    """float64 autograd of conv2d (+SiLU): (dx [B*h*w, cin], dW OIHW, dbias)"""
    with torch.enable_grad():  # other tests switch autograd off process-wide
        x64 = x.double().view(batch, h, w, cin).permute(0, 3, 1, 2).contiguous().requires_grad_()
        w64 = wp.double().requires_grad_()
        b64 = (b.double() if b is not None else torch.zeros(cout, dtype=torch.float64, device=x.device)).requires_grad_()
        y = F.conv2d(x64, w64, b64, stride=stride, padding=1)
        if silu:
            y = F.silu(y)
        (y * dy.double().view(batch, ho, wo, cout).permute(0, 3, 1, 2)).sum().backward()
    return x64.grad.permute(0, 2, 3, 1).reshape(batch * h * w, cin), w64.grad, b64.grad


def case_conv_bwd(batch, h, w, cin, cout, stride=1, silu=False, bias=True, grads=("x", "w", "bias"), accumulate=(),
                  seed=0):
    """conv3x3_direct_backward of one layer; accumulate: dW / dbias added onto random destinations"""
    x, wp, wt, b, dy, ho, wo = _conv_inputs(batch, h, w, cin, cout, stride, bias, seed)
    outs = {}
    if "x" in grads:
        outs["x"] = Guarded(batch * h * w, cin, contiguous=True)
    if "w" in grads:
        outs["w"] = Guarded(cout, 9 * cin, torch.float32, contiguous=True, shape=(cout, cin, 3, 3))
    if "bias" in grads:
        outs["bias"] = Guarded(1, cout, torch.float32, contiguous=True, shape=(cout,))
    init = {}
    for i, nm in enumerate(accumulate):
        init[nm] = _rand(*outs[nm].out.shape, seed=seed + 10 + i)
        outs[nm].out.copy_(init[nm])
    dx, dw, db = ops.conv3x3_direct_backward(
        x, wt, dy, batch=batch, h=h, w=w, cin=cin, cout=cout, stride=stride, bias=b, silu=silu, grads=grads,
        accumulate=accumulate, **{f"out_d{nm}": g.out for nm, g in outs.items()})
    for nm, g in outs.items():
        g.check("d" + nm)
    rx, rw, rb = _conv_ref(x, wp, b, dy, batch, h, w, cin, cout, stride, silu, ho, wo)
    errs, tols, note = {}, {}, ""
    if dx is not None:
        errs["dx"], note = gated(dx, rx, TOL)
        tols["dx"] = TOL
    for nm, got, ref in (("w", dw, rw), ("bias", db, rb)):
        if got is not None:
            base = init.get(nm)
            errs["d" + nm] = rel(got, ref if base is None else base.double() + ref)
            tols["d" + nm] = TOL_F32
    desc = (f"direct conv backward B={batch} {h}x{w} {cin}->{cout} s{stride} silu={silu} bias={bias} "
            f"grads={','.join(grads)} acc={','.join(accumulate)}")
    return _gate(errs, tols, desc + note)


def case_conv_ad(batch, h, w, cin, cout, stride=1, silu=True, residual=True, seed=0):
    """the autograd op direct_conv3x3: the residual's gradient is dy bit for bit, the forward output is the inference
    kernel's, and x / w_param / bias get their gradients"""
    x, wp, wt, b, dy, ho, wo = _conv_inputs(batch, h, w, cin, cout, stride, True, seed)
    res = _rand(batch * ho * wo, cout, seed=seed + 5).half() if residual else None
    kw = dict(batch=batch, h=h, w=w, cin=cin, cout=cout, stride=stride, silu=silu)
    with torch.enable_grad():
        xs = x.clone().requires_grad_()
        wl, bl = wp.clone().requires_grad_(), b.clone().requires_grad_()
        rl = res.clone().requires_grad_() if residual else None
        y = ops.direct_conv3x3(xs, wt, w_param=wl, bias=bl, residual=rl, **kw)
        y.backward(dy)
    assert torch.equal(y, ops.conv3x3_direct(x, wt, b, residual=res, **kw)), "forward differs from the inference path"
    if residual:
        assert torch.equal(rl.grad, dy), "the residual's gradient must be dy"
    rx, rw, rb = _conv_ref(x, wp, b, dy, batch, h, w, cin, cout, stride, silu, ho, wo)
    errs = {"dx": rel(xs.grad, rx), "dw": rel(wl.grad, rw), "dbias": rel(bl.grad, rb)}
    tols = {"dx": TOL, "dw": TOL_F32, "dbias": TOL_F32}
    return _gate(errs, tols, f"direct_conv3x3 autograd B={batch} {h}x{w} {cin}->{cout} s{stride} silu={silu} "
                             f"residual={residual}")


def case_skinny_bwd(rows, n, k, silu_in, accumulate=(), seed=0):
    """skinny_linear_backward; rows > 16 runs in row chunks"""
    x = _rand(rows, k, seed=seed)
    wp = _rand(n, k, seed=seed + 1, scale=k ** -0.5).half()
    dy = _rand(rows, n, seed=seed + 2)
    g = {"x": Guarded(rows, k, torch.float32, contiguous=True), "w": Guarded(n, k, torch.float32, contiguous=True),
         "bias": Guarded(1, n, torch.float32, contiguous=True, shape=(n,))}
    init = {}
    for i, nm in enumerate(accumulate):
        init[nm] = _rand(*g[nm].out.shape, seed=seed + 10 + i)
        g[nm].out.copy_(init[nm])
    dx, dw, db = ops.skinny_linear_backward(x, wp, dy, silu_in=silu_in, out_dx=g["x"].out, out_dw=g["w"].out,
                                            out_dbias=g["bias"].out, accumulate=accumulate)
    for nm, gg in g.items():
        gg.check("d" + nm)
    with torch.enable_grad():
        x64, w64 = x.double().requires_grad_(), wp.double().requires_grad_()
        b64 = torch.zeros(n, dtype=torch.float64, device=x.device, requires_grad=True)
        (F.linear(F.silu(x64) if silu_in else x64, w64, b64) * dy.double()).sum().backward()
    errs = {}
    for nm, got, ref in (("x", dx, x64.grad), ("w", dw, w64.grad), ("bias", db, b64.grad)):
        base = init.get(nm)
        errs["d" + nm] = rel(got, ref if base is None else base.double() + ref)
    return _gate(errs, dict.fromkeys(errs, TOL_F32),
                 f"skinny backward rows={rows} n={n} k={k} silu_in={silu_in} acc={','.join(accumulate)}")


def case_upsample_bwd(batch, h, w, c, dx_dtype="f16", accumulate=False, seed=0):
    dt = {"f16": torch.float16, "f32": torch.float32}[dx_dtype]
    dy = _rand(batch * 4 * h * w, c, seed=seed).half()
    g = Guarded(batch * h * w, c, dt, contiguous=True)
    base = None
    if accumulate:
        base = _rand(batch * h * w, c, seed=seed + 1).to(dt)
        g.out.copy_(base)
    dx = ops.upsample2x_backward(dy, batch=batch, h=h, w=w, c=c, out_dx=g.out, accumulate=accumulate)
    g.check("dx")
    with torch.enable_grad():
        x64 = torch.zeros(batch, c, h, w, dtype=torch.float64, device=dy.device, requires_grad=True)
        up = F.interpolate(x64, scale_factor=2, mode="nearest")
        (up * dy.double().view(batch, 2 * h, 2 * w, c).permute(0, 3, 1, 2)).sum().backward()
    ref = x64.grad.permute(0, 2, 3, 1).reshape(batch * h * w, c)
    if base is not None:
        ref = ref + base.double()
    err = rel(dx, ref)
    return err, TOL if dt == torch.float16 else TOL_F32, (f"upsample2x backward B={batch} {h}x{w} c={c} "
                                                          f"dx={dx_dtype} acc={accumulate}: rel-L2 {err:.2e}")


CASES = []
# every hint layer at 512^2 (B = 1) and 128^2 (B = 2) pose maps; the first layer's input is the pose map (no dx)
for _s, _b in ((512, 1), (128, 2)):
    for _cin, _cout, _st, _div in HINT_LAYERS:
        CASES.append((case_conv_bwd, dict(batch=_b, h=_s // _div, w=_s // _div, cin=_cin, cout=_cout, stride=_st,
                                          silu=True, grads=("w", "bias") if _cin == 3 else ("x", "w", "bias"))))
# conv_in 4 -> 320 (transpose 320 -> 4: the small-cout kernel) and out 320 -> 4 (transpose 4 -> 320: small-cin)
for _hw in (64, 16):
    for _b in (1, 2, 4):
        CASES.append((case_conv_bwd, dict(batch=_b, h=_hw, w=_hw, cin=4, cout=320)))
        CASES.append((case_conv_bwd, dict(batch=_b, h=_hw, w=_hw, cin=320, cout=4)))
CASES += [
    # ragged channel counts, odd and non-square images, stride 2 on odd sizes
    (case_conv_bwd, dict(batch=2, h=7, w=5, cin=3, cout=3)),
    (case_conv_bwd, dict(batch=2, h=7, w=5, cin=3, cout=8, stride=2, silu=True)),
    (case_conv_bwd, dict(batch=1, h=12, w=8, cin=16, cout=3, silu=True)),
    (case_conv_bwd, dict(batch=3, h=33, w=31, cin=3, cout=16, stride=2, silu=True)),
    (case_conv_bwd, dict(batch=2, h=33, w=31, cin=16, cout=8)),
    (case_conv_bwd, dict(batch=2, h=33, w=31, cin=8, cout=16, stride=2)),
    (case_conv_bwd, dict(batch=1, h=12, w=8, cin=32, cout=96, stride=2, silu=True)),
    (case_conv_bwd, dict(batch=2, h=33, w=31, cin=40, cout=24, silu=True, bias=False)),
    # one gradient at a time, and accumulation into dW / dbias
    (case_conv_bwd, dict(batch=2, h=32, w=32, cin=16, cout=32, stride=2, silu=True, grads=("x",))),
    (case_conv_bwd, dict(batch=2, h=32, w=32, cin=16, cout=32, silu=True, grads=("bias",))),
    (case_conv_bwd, dict(batch=2, h=32, w=32, cin=16, cout=32, silu=True, accumulate=("w", "bias"))),
    # the autograd op: SiLU on and off, with and without a residual
    (case_conv_ad, dict(batch=2, h=32, w=32, cin=16, cout=32, silu=True, residual=False)),
    (case_conv_ad, dict(batch=2, h=16, w=16, cin=4, cout=320, silu=False, residual=True)),
    (case_conv_ad, dict(batch=2, h=33, w=31, cin=32, cout=96, stride=2, silu=True, residual=True)),
]
# the stacked emb_layers of the UNet / appearance net (20160 rows) and of the pose net (9600), and time_embed.0 / .2
for _n in (20160, 9600):
    for _rows in (1, 2, 4, 20):
        for _silu in (True, False):
            CASES.append((case_skinny_bwd, dict(rows=_rows, n=_n, k=1280, silu_in=_silu)))
CASES += [
    (case_skinny_bwd, dict(rows=4, n=1280, k=320, silu_in=False)),
    (case_skinny_bwd, dict(rows=4, n=1280, k=1280, silu_in=True)),
    (case_skinny_bwd, dict(rows=20, n=1280, k=1280, silu_in=True, accumulate=("x", "w", "bias"))),
]
for _hw in (8, 32):
    for _c in (1280, 640):
        CASES.append((case_upsample_bwd, dict(batch=2, h=_hw, w=_hw, c=_c)))
CASES += [
    (case_upsample_bwd, dict(batch=2, h=16, w=16, c=640, dx_dtype="f32")),
    (case_upsample_bwd, dict(batch=2, h=16, w=16, c=640, dx_dtype="f32", accumulate=True)),
    (case_upsample_bwd, dict(batch=1, h=7, w=5, c=320, accumulate=True)),
]


def case_id(case):
    fn, kw = case
    return fn.__name__.removeprefix("case_") + "-" + "-".join(f"{k}={v}" for k, v in kw.items()).replace(
        " ", "").replace("'", "")
