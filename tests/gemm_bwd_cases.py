"""Numerics cases of the GEMM / implicit-GEMM convolution backward (ops.gemm_backward): each case runs the backward on
the GPU and returns (error, tolerance, description) against torch fp32 autograd of F.linear / F.conv2d computed from
the SAME fp16-rounded inputs.  Run by tests/test_gemm_bwd_gpu.py; the same (error, tolerance, description) contract
as tests/kernel_cases.py.  The error is the largest over the requested gradients of the rel-L2, gated per 128 x 32
block for dA, dA2 and dW (tests/kernel_guard.py).

Every gradient goes into a NaN-poisoned, guarded buffer, so an element that is never written, or a write outside the
gradient, fails the case; the row-stride padding of dd, a, a2 and w holds NaN; the "gemm_bwd" workspace holds NaN
before each call; and every case runs twice and requires bit-equal gradients (the split reductions are summed in a
fixed order)."""
import torch
import torch.nn.functional as F

from magicdance_b200 import ops
from tests.kernel_cases import DEV, _rand, nan_padded
from tests.kernel_guard import Guarded, bit_equal, check_workspace_used, gated, poison_workspace, rel

TOL = 2e-3  # the forward GEMM's gate
_DT = {"f16": torch.float16, "f32": torch.float32}


def _run(a, w, dd, kw, specs, init, desc):
    """one gemm_backward into Guarded destinations (specs: {name: (rows, cols, dtype, contiguous, shape)}, names in
    init start from those contents), against a poisoned workspace; returns {name: gradient}"""
    outs = {nm: Guarded(r, c, dt, contiguous=cont, shape=shape) for nm, (r, c, dt, cont, shape) in specs.items()}
    for nm, t in init.items():
        outs[nm].out.copy_(t)
    ws = poison_workspace("gemm_bwd", device=a.device)
    ops.gemm_backward(a, w, dd, **kw, **{f"out_d{nm}": g.out for nm, g in outs.items()})
    for nm, g in outs.items():
        g.check(f"{desc} d{nm}")
    return {nm: g.out for nm, g in outs.items()}, ws


def case_gemm_bwd(m, n, k, conv=None, stride=1, k2=0, bias=None, rows_per_batch=0, grads=("a", "b"), da_dtype="f16",
                  db_dtype="f32", accumulate=(), splits=0, db_splits=0, seed=0):
    """m, n, k: the forward's M x N x K (conv=(nb, h, w): k = 9c, m is derived); k2: columns of a second source a2;
    bias: None | "row" | "batch" (per segment of rows_per_batch rows); accumulate: gradients added into random
    destinations."""
    if conv is not None:
        nb, h, w_ = conv
        c = k // 9
        ho, wo = (h - 1) // stride + 1, (w_ - 1) // stride + 1
        m = nb * ho * wo
        a = _rand(nb * h * w_, c, seed=seed).half()  # the conv path takes a dense NHWC activation
        a2 = None
    else:
        a = nan_padded(_rand(m, k - k2, seed=seed).half())
        a2 = nan_padded(_rand(m, k2, seed=seed + 4).half()) if k2 else None
    w = nan_padded(_rand(n, k, seed=seed + 1, scale=k ** -0.5).half())
    dd = nan_padded(_rand(m, n, seed=seed + 2).half())
    grads = tuple(grads) + (("bias",) if bias else ())
    kw = dict(a2=a2, splits=splits, db_splits=db_splits, grads=grads, accumulate=accumulate)
    if conv is not None:
        kw.update(conv=(nb, h, w_, c), conv_stride=stride)
    segs = 1
    if bias == "batch":
        segs = -(-m // rows_per_batch)
        kw.update(bias_batch_stride=n, rows_per_batch=rows_per_batch)
    specs = {}
    if "a" in grads:
        specs["a"] = (*a.shape, _DT[da_dtype], False, None)
        if a2 is not None:
            specs["a2"] = (m, k2, _DT[da_dtype], False, None)
    if "b" in grads:
        specs["b"] = (n, k, _DT[db_dtype], False, None)
    if "bias" in grads:
        specs["bias"] = (segs, n, torch.float32, True, (n,) if bias == "row" else (segs, n))
    # destinations to accumulate into start from random contents
    init = {}
    if "a" in accumulate:
        init["a"] = _rand(*a.shape, seed=seed + 5).to(_DT[da_dtype])
    if "b" in accumulate:
        init["b"] = _rand(n, k, seed=seed + 6).to(_DT[db_dtype])
    if "bias" in accumulate:
        init["bias"] = _rand(*((n,) if bias == "row" else (segs, n)), seed=seed + 7).float()
    shape = f"conv{stride} nb={conv[0]} {conv[1]}x{conv[2]} {c}->{n}" if conv is not None else f"m={m} n={n} k={k}"
    desc = (f"gemm backward {shape} k2={k2} bias={bias} rpb={rows_per_batch} da={da_dtype} db={db_dtype} "
            f"acc={','.join(accumulate)} splits={splits}/{db_splits}")
    got, _ = _run(a, w, dd, kw, specs, init, desc)
    again, ws = _run(a, w, dd, kw, specs, init, desc + " (second run)")
    check_workspace_used("gemm_bwd", ws, desc, a.device)
    for nm in got:
        if not bit_equal(got[nm], again[nm]):
            raise AssertionError(f"{desc}: d{nm} differs between two runs")

    with torch.enable_grad():  # other tests switch autograd off process-wide
        wf = w.float().requires_grad_()
        if conv is not None:
            xf = a.float().view(nb, h, w_, c).permute(0, 3, 1, 2).contiguous().requires_grad_()
            wc = wf.view(n, 3, 3, c).permute(0, 3, 1, 2)
            out = F.conv2d(xf, wc, stride=stride, padding=1).permute(0, 2, 3, 1).reshape(m, n)
            inputs = [xf]
        else:
            af = a.float().requires_grad_()
            a2f = a2.float().requires_grad_() if a2 is not None else None
            out = F.linear(torch.cat([af, a2f], 1) if a2 is not None else af, wf)
            inputs = [af] + ([a2f] if a2 is not None else [])
        (out * dd.float()).sum().backward()
    ddf = dd.float()
    refs = {}
    if conv is not None:
        refs["a"] = xf.grad.permute(0, 2, 3, 1).reshape(nb * h * w_, c)
    else:
        refs["a"] = inputs[0].grad
        if a2 is not None:
            refs["a2"] = inputs[1].grad
    refs["b"] = wf.grad
    if bias == "row":
        refs["bias"] = ddf.sum(0)
    elif bias == "batch":
        refs["bias"] = torch.stack([ddf[s * rows_per_batch:(s + 1) * rows_per_batch].sum(0) for s in range(segs)])
    errs, notes = {}, ""
    for name, ref in refs.items():
        if name not in got:
            continue
        base = init.get(name)
        ref = ref if base is None else base.float() + ref
        if name == "bias":
            errs[name] = rel(got[name].float(), ref)
        else:
            errs[name], note = gated(got[name].float(), ref, TOL)
            notes += f" d{name}{note}"
    desc += ": error " + " ".join(f"d{nm} {e:.2e}" for nm, e in errs.items()) + notes
    return max(errs.values()), TOL, desc


# keyword arguments of case_gemm_bwd; config-5 sizes are batch 4 at a 64x64 latent
CASES = [
    # Linear at 64x64 x batch 4 (M = 16384 tokens)
    dict(m=16384, n=320, k=320, bias="row"),                 # attn q/k/v/out, proj_in/out
    dict(m=16384, n=2560, k=320),                            # GEGLU proj (dD = the pre-activation gradient)
    dict(m=16384, n=320, k=1280),                            # FF out
    dict(m=1024, n=1280, k=1280, bias="row"),
    # text projections to_k / to_v of the cross-attention: 4 x 77 tokens, K = 768, weight gradient only
    dict(m=308, n=320, k=768, grads=("b",)),
    dict(m=308, n=1280, k=768, grads=("b",)),
    # ragged M
    dict(m=1000, n=320, k=640, bias="row"),
    # the V^T form gemm(W_v, x): dA is the weight gradient (fp32, reduces over tokens), dB the activation's (fp16)
    dict(m=320, n=4096, k=320, da_dtype="f32", db_dtype="f16"),
    dict(m=320, n=77, k=768, da_dtype="f32", db_dtype="f16"),  # text V^T: N = 77
    # dual source: 640 + 320 channels of the skip concat -> 320
    dict(m=4096, n=320, k=960, k2=320, bias="row"),
    # per-batch bias (timestep embedding), 4 segments
    dict(m=4096, n=640, k=640, bias="batch", rows_per_batch=1024),
    # accumulate into the destination
    dict(m=2048, n=320, k=320, accumulate=("a",)),
    dict(m=2048, n=320, k=320, bias="row", da_dtype="f32", accumulate=("a", "b", "bias")),
    # forced splits of both reductions: counts the automatic choice does not take, and none
    dict(m=1024, n=1280, k=1280, splits=3, db_splits=5),
    dict(m=1024, n=1280, k=1280, splits=1, db_splits=1),
    dict(m=0, n=320, k=9 * 320, conv=(1, 32, 32), splits=2, db_splits=3),
    dict(m=0, n=320, k=9 * 320, conv=(1, 32, 32), splits=1, db_splits=1),
]
for _nb in (1, 4):  # 3x3 stride 1 (implicit dA and dB)
    CASES += [
        dict(m=0, n=320, k=9 * 320, conv=(_nb, 64, 64), bias="row"),
        dict(m=0, n=640, k=9 * 640, conv=(_nb, 32, 32)),
        dict(m=0, n=1280, k=9 * 1280, conv=(_nb, 16, 16)),
        dict(m=0, n=1280, k=9 * 1280, conv=(_nb, 8, 8)),
        dict(m=0, n=1280, k=9 * 2560, conv=(_nb, 8, 8)),
        dict(m=0, n=320, k=9 * 960, conv=(_nb, 64, 64)),
    ]
CASES += [
    # 3x3 stride 2 (Downsample): dA through the column buffer, dB implicit with TMA element strides
    dict(m=0, n=320, k=9 * 320, conv=(2, 64, 64), stride=2, bias="row"),
    dict(m=0, n=640, k=9 * 640, conv=(2, 32, 32), stride=2),
    dict(m=0, n=1280, k=9 * 1280, conv=(2, 16, 16), stride=2),
    # a 12x8 latent does not tile into the TMA boxes: column path for dA, im2col for dB
    dict(m=0, n=320, k=9 * 320, conv=(2, 12, 8), bias="row"),
    dict(m=0, n=320, k=9 * 320, conv=(2, 12, 8), stride=2),
]
CASES += [
    # ragged M: one row, one 64-row half tile, one row short of and past a 128-row tile
    *(dict(m=_m, n=320, k=320, bias="row") for _m in (1, 64, 127, 129)),
    # the token counts of a 40x24 latent's four levels at batch 2 (15 / 60 / 240 / 960 tokens per sample)
    *(dict(m=_m, n=320, k=640, bias="row") for _m in (30, 120, 480, 1920)),
    # N tails: dA reduces over N, dW and dbias have N rows
    *(dict(m=1000, n=_n, k=320, bias="row") for _n in (8, 72, 77, 200)),
    # K of one 64-wide chunk, and 192: half of the last 128-wide dA / dW column tile
    dict(m=1000, n=320, k=64, bias="row"),
    dict(m=1000, n=320, k=192),
    # the output blocks' 320 + 320 skip concat: the split between a and a2 falls inside a 128-wide tile
    dict(m=4096, n=320, k=640, k2=320, bias="row"),
    dict(m=1000, n=320, k=640, k2=320, splits=3, db_splits=5),
    # forced splits that leave the last one short, of both reductions
    dict(m=1000, n=1160, k=640, splits=7, db_splits=11),
    dict(m=0, n=640, k=9 * 320, conv=(2, 12, 8), splits=3, db_splits=5),
    # per-batch bias over segments shorter than one 128-row tile (a 40x24 latent's deep levels)
    dict(m=480, n=320, k=320, bias="batch", rows_per_batch=60),
    dict(m=60, n=1280, k=1280, bias="batch", rows_per_batch=15),
    dict(m=308, n=320, k=320, bias="batch", rows_per_batch=77),
    # the TMA-box conv path at the deepest level with an odd batch, and at 4x4
    dict(m=0, n=1280, k=9 * 1280, conv=(3, 8, 8), bias="row"),
    dict(m=0, n=1280, k=9 * 1280, conv=(2, 4, 4)),
    dict(m=0, n=640, k=9 * 1280, conv=(4, 4, 4), bias="row"),
]


def case_id(kw):
    return "-".join(f"{k}={v}" for k, v in kw.items()).replace(" ", "").replace("'", "")
