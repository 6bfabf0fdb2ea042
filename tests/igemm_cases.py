"""Numerics cases of the 3x3 convolution at any latent size (ops.conv3x3_igemm / conv3x3_igemm_backward: TMA im2col
loads into the wgmma GEMM and its backward).  Each case runs on the GPU into sentinel-filled outputs (tests/kernel_guard)
and returns (error, tolerance, description) against torch fp32 F.conv2d and its autograd gradients computed from the
SAME fp16-rounded inputs, like tests/kernel_cases.py.  Run by tests/test_conv_igemm_gpu.py."""
import torch
import torch.nn.functional as F

from magicdance_b200 import ops
from tests.kernel_cases import DEV, _rand
from tests.kernel_guard import Guarded, gated, rel

TOL = 2e-3  # the box-path conv's gate (tests/kernel_cases.py, tests/gemm_bwd_cases.py)


def _strided(t, pad):
    """t [pixels, c] as the first c columns of a [pixels, c + pad] buffer (a pixel stride other than c) whose other
    columns hold NaN"""
    if not pad:
        return t
    buf = torch.full((t.shape[0], t.shape[1] + pad), float("nan"), dtype=t.dtype, device=t.device)
    buf[:, :t.shape[1]] = t
    return buf[:, :t.shape[1]]


def _inputs(nb, h, w, cin, cout, c2, seed, pad=0):
    c1 = cin - c2
    x = _strided(_rand(nb * h * w, c1, seed=seed).half(), pad)
    x2 = _strided(_rand(nb * h * w, c2, seed=seed + 1).half(), pad) if c2 else None
    wt = _rand(cout, 9 * cin, seed=seed + 2, scale=(9 * cin) ** -0.5).half()  # [O][kh][kw][I]
    return x, x2, wt


def _nchw(x, x2, nb, h, w):
    xs = x.float() if x2 is None else torch.cat([x.float(), x2.float()], 1)
    return xs.reshape(nb, h, w, -1).permute(0, 3, 1, 2)


def _oihw(wt, cin):
    return wt.float().reshape(wt.shape[0], 3, 3, cin).permute(0, 3, 1, 2)


def case_fwd(nb, h, w, cin, cout, stride=1, c2=0, bias=None, residual=False, splits=0, pad=0, seed=0):
    """y = conv3x3(x [; x2]) (+ bias row | per-image bias) (+ residual) into a guarded [M, cout] output; pad: the
    sources' pixel stride exceeds their channels by `pad` NaN columns"""
    x, x2, wt = _inputs(nb, h, w, cin, cout, c2, seed, pad)
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    m = nb * ho * wo
    kw = dict(conv=(nb, h, w, cin), conv_stride=stride, x2=x2, splits=splits)
    ref = F.conv2d(_nchw(x, x2, nb, h, w), _oihw(wt, cin), padding=1, stride=stride).permute(0, 2, 3, 1).reshape(m, cout)
    if bias == "row":
        b = _rand(cout, seed=seed + 3).float()
        kw.update(bias=b)
        ref = ref + b
    elif bias == "batch":
        b = _rand(nb, cout, seed=seed + 3).float()
        kw.update(bias=b, bias_batch_stride=cout, rows_per_batch=ho * wo)
        ref = ref + b.repeat_interleave(ho * wo, 0)
    if residual:
        r = _rand(m, cout, seed=seed + 4).half()
        kw.update(residual=r)
        ref = ref + r.float()
    g = Guarded(m, cout)
    y = ops.conv3x3_igemm(x, wt, out=g.out, **kw)
    desc = (f"igemm fwd B={nb} {h}x{w} {cin}->{cout} s={stride} c2={c2} bias={bias} res={residual} splits={splits} "
            f"pad={pad}")
    g.check(desc)
    err, note = gated(y, ref, TOL)
    return err, TOL, desc + note


def case_bwd(nb, h, w, cin, cout, stride=1, c2=0, bias=None, splits=0, db_splits=0, pad=0, seed=0):
    """dx (fp16, and dx2 with a second source), dW (fp32) and dbias of the conv against torch autograd, every output
    in a guarded buffer; pad as in case_fwd"""
    x, x2, wt = _inputs(nb, h, w, cin, cout, c2, seed, pad)
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    m = nb * ho * wo
    dd = _rand(m, cout, seed=seed + 5).half()
    xr = _nchw(x, x2, nb, h, w).requires_grad_()
    wr = _oihw(wt, cin).requires_grad_()
    y = F.conv2d(xr, wr, padding=1, stride=stride).permute(0, 2, 3, 1).reshape(m, cout)
    y.backward(dd.float())
    gx = xr.grad.permute(0, 2, 3, 1).reshape(nb * h * w, cin)
    gw = wr.grad.permute(0, 2, 3, 1).reshape(cout, 9 * cin)
    kw = dict(conv=(nb, h, w, cin), conv_stride=stride, x2=x2, splits=splits, db_splits=db_splits,
              grads=("a", "b") + (("bias",) if bias else ()))
    if bias == "batch":
        kw.update(bias_batch_stride=cout, rows_per_batch=ho * wo)
        gb = dd.float().reshape(nb, ho * wo, cout).sum(1)
    else:
        gb = dd.float().sum(0)
    if bias:
        gdb = Guarded(nb if bias == "batch" else 1, cout, torch.float32, contiguous=True, shape=tuple(gb.shape))
        kw.update(out_dbias=gdb.out)
    gda = Guarded(nb * h * w, cin - c2)
    gdw = Guarded(cout, 9 * cin, torch.float32)
    kw.update(out_da=gda.out, out_db=gdw.out)
    if c2:
        gda2 = Guarded(nb * h * w, c2)
        kw.update(out_da2=gda2.out)
    dx, dx2, dw, dbias = ops.conv3x3_igemm_backward(x, wt, dd, **kw)
    desc = (f"igemm bwd B={nb} {h}x{w} {cin}->{cout} s={stride} c2={c2} bias={bias} splits={splits}/{db_splits} "
            f"pad={pad}")
    gda.check(desc + " dx")
    if bias:
        gdb.check(desc + " dbias")
    gdw.check(desc + " dW")
    if c2:
        gda2.check(desc + " dx2")
        dx = torch.cat([dx.float(), dx2.float()], 1)
    e_x, n_x = gated(dx, gx, TOL)
    e_w, n_w = gated(dw, gw, TOL)
    errs = [e_x, e_w]
    if bias:
        errs.append(rel(dbias, gb))
    return max(errs), TOL, desc + f" dx{n_x} dW{n_w}"


FWD_CASES = [
    # every level of a 40x24 latent (none tiles) and the non-tiling levels of 112x64 and 96x64
    dict(nb=2, h=40, w=24, cin=320, cout=320, bias="batch"),
    dict(nb=2, h=20, w=12, cin=640, cout=640, bias="batch", residual=True),
    dict(nb=2, h=10, w=6, cin=1280, cout=1280, bias="batch"),
    dict(nb=2, h=5, w=3, cin=2560, cout=1280, c2=1280, bias="batch", residual=True),
    dict(nb=1, h=28, w=16, cin=640, cout=640, bias="row", residual=True),
    dict(nb=1, h=14, w=8, cin=1280, cout=1280),
    dict(nb=1, h=112, w=64, cin=320, cout=320, bias="batch", residual=True),
    dict(nb=16, h=12, w=8, cin=1280, cout=1280, bias="batch"),
    dict(nb=16, h=5, w=3, cin=1280, cout=1280, residual=True),
    # dual source (fused skip concat) at every channel split the UNet's output blocks have
    dict(nb=2, h=14, w=8, cin=1920, cout=640, c2=640, bias="batch"),
    dict(nb=2, h=28, w=16, cin=960, cout=320, c2=320, residual=True),
    dict(nb=2, h=10, w=6, cin=640, cout=320, c2=320),
    # stride 2 (Downsample), odd and even sides
    dict(nb=2, h=40, w=24, cin=320, cout=320, stride=2, bias="row"),
    dict(nb=2, h=10, w=6, cin=1280, cout=1280, stride=2, bias="row"),
    dict(nb=1, h=112, w=64, cin=320, cout=320, stride=2, bias="row"),
    dict(nb=1, h=28, w=16, cin=640, cout=640, stride=2),
    dict(nb=16, h=5, w=3, cin=640, cout=640, stride=2),
    # forced split-K: cluster (2, 4, 8) and workspace (3) reductions, with the epilogue operands
    dict(nb=2, h=5, w=3, cin=1280, cout=1280, splits=2, bias="batch", residual=True),
    dict(nb=2, h=10, w=6, cin=1280, cout=1280, splits=4, bias="row"),
    dict(nb=1, h=14, w=8, cin=2560, cout=1280, c2=1280, splits=8, residual=True),
    dict(nb=2, h=12, w=8, cin=640, cout=640, splits=3, bias="batch", residual=True),
    # pixel strides wider than the channels (lda, lda2 > c)
    dict(nb=2, h=20, w=12, cin=640, cout=640, pad=64, bias="row"),
    dict(nb=2, h=14, w=8, cin=1920, cout=640, c2=640, pad=8, residual=True),
    dict(nb=2, h=40, w=24, cin=320, cout=320, stride=2, pad=16),
    # ragged N tiles and a 77-wide output
    dict(nb=2, h=12, w=8, cin=320, cout=200),
    dict(nb=2, h=10, w=6, cin=64, cout=77, bias="row"),
]

BWD_CASES = [
    dict(nb=2, h=40, w=24, cin=320, cout=320, bias="batch"),
    dict(nb=2, h=20, w=12, cin=640, cout=640),
    dict(nb=2, h=10, w=6, cin=1280, cout=1280, bias="batch"),
    dict(nb=2, h=5, w=3, cin=2560, cout=1280, c2=1280, bias="batch"),
    dict(nb=1, h=28, w=16, cin=640, cout=640, bias="row"),
    dict(nb=1, h=14, w=8, cin=1280, cout=1280),
    dict(nb=1, h=112, w=64, cin=320, cout=320, bias="batch"),
    dict(nb=16, h=12, w=8, cin=1280, cout=1280),
    dict(nb=16, h=5, w=3, cin=640, cout=640, bias="batch"),
    dict(nb=2, h=14, w=8, cin=1920, cout=640, c2=640),
    dict(nb=2, h=40, w=24, cin=320, cout=320, stride=2, bias="row"),
    dict(nb=1, h=112, w=64, cin=320, cout=320, stride=2),
    dict(nb=2, h=10, w=6, cin=1280, cout=1280, stride=2),
    dict(nb=16, h=5, w=3, cin=640, cout=640, stride=2),
    dict(nb=2, h=10, w=6, cin=1280, cout=1280, splits=3, db_splits=5),
    dict(nb=2, h=12, w=8, cin=640, cout=200, splits=1, db_splits=1),
    dict(nb=2, h=20, w=12, cin=640, cout=640, pad=64, bias="row"),
    dict(nb=2, h=14, w=8, cin=1920, cout=640, c2=640, pad=8, bias="batch"),
    dict(nb=2, h=40, w=24, cin=320, cout=320, stride=2, pad=16),
]


def case_id(kw):
    return "-".join(f"{k}{v}" for k, v in kw.items())


def box_vs_im2col(nb, h, w, cin, cout, stride, seed=0):
    """(forward, backward) of the box path (ops.gemm / gemm_backward with conv=...) and of the im2col path at a size
    both take: bit-equal, since both feed the same swizzled tiles to the same wgmma in the same K order"""
    x, _, wt = _inputs(nb, h, w, cin, cout, 0, seed)
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    m = nb * ho * wo
    b = _rand(nb, cout, seed=seed + 3).float()
    r = _rand(m, cout, seed=seed + 4).half()
    dd = _rand(m, cout, seed=seed + 5).half()
    conv = (nb, h, w, cin)
    fk = dict(bias=b, bias_batch_stride=cout, rows_per_batch=ho * wo, residual=r)
    y_box = ops.gemm(x, wt, conv=conv, conv_stride=stride, **fk)
    y_im = ops.conv3x3_igemm(x, wt, conv=conv, conv_stride=stride, **fk)
    bk = dict(conv=conv, conv_stride=stride, bias_batch_stride=cout, rows_per_batch=ho * wo, grads=("a", "b", "bias"))
    g_box = ops.gemm_backward(x, wt, dd, **bk)
    g_im = ops.conv3x3_igemm_backward(x, wt, dd, **bk)
    return (y_box, y_im), [(p, q) for p, q in zip(g_box, g_im) if p is not None]
