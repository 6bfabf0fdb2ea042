"""TEST DOUBLES — differentiable PyTorch (CPU) stand-ins for the autograd ops of `magicdance_b200.ops` that the training
forward (magicdance_b200/train.py) calls.  They read the same packed layouts as the kernels (NHWC fp16 activations
[B*H*W, C]; conv weights [O][kh][kw][I]; 1x1 / linear weights [O, I]; V^T by swapped operands), round every activation
to fp16 like the kernels, and take each weight term from the fp32 tensor passed beside its fp16 copy (w_param /
a_param) — with the copy's values — so that gradients land in the parameters' own layouts.  Each asserts that the copy
equals that tensor packed, which catches layout mistakes and stale copies.  Never imported by the product."""
import torch
import torch.nn.functional as F

from tests import fake_ops

PATCHED = ("tc_gemm", "two_source_attention", "group_norm", "layer_norm", "geglu", "direct_conv3x3", "skinny_linear_ad",
           "upsample_2x", "add_ad", "nchw_to_nhwc", "nhwc_to_nchw", "timestep_embedding", "ensure_device",
           "require_cuda")


def _h(t):
    return t.to(torch.float16)


def _conv_packed(w):
    """Conv2d OIHW -> [O][kh][kw][I] as [O, 9*I]; a matrix as it is"""
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1) if w.dim() == 4 else w


def _unpack(copy16, shape):
    """a [O][kh][kw][I] copy back in the OIHW layout"""
    o, i, kh, kw = shape
    return copy16.float().reshape(o, kh, kw, i).permute(0, 3, 1, 2)


def _weight(copy16, param):
    """param with the value the kernel sees (copy16, which must equal param packed and rounded to fp16) and param's
    gradient"""
    assert copy16.dtype == torch.float16
    want = _conv_packed(param.detach()).to(torch.float16)
    assert copy16.shape == want.shape and torch.equal(copy16, want), "fp16 copy differs from its parameter packed"
    value = _unpack(copy16, param.shape) if param.dim() == 4 else copy16.float()
    return param + (value - param).detach()


def tc_gemm(a, w, *, a_param=None, w_param=None, bias=None, bias_batch_stride=0, rows_per_batch=0, residual=None,
            a2=None, conv=None, conv_stride=1, splits=0, m=None, epilogue=0, ln_u=None):
    assert epilogue == 0 and ln_u is None, "no backward exists for the fused epilogues"
    assert a.dtype == torch.float16 and w.dtype == torch.float16
    A = _weight(a, a_param) if a_param is not None else a.float()
    n, k = w.shape
    if conv is not None:
        b, h, ww, cin = conv
        assert a2 is None and k == 9 * cin
        if w_param is not None:
            assert w_param.dim() == 4
            W = _weight(w, w_param)
        else:
            W = w.float().reshape(n, 3, 3, cin).permute(0, 3, 1, 2)
        x = A.reshape(b, h, ww, cin).permute(0, 3, 1, 2)
        y = F.conv2d(x, W, None, padding=1, stride=conv_stride).permute(0, 2, 3, 1).reshape(-1, n)
    else:
        W = _weight(w, w_param) if w_param is not None else w.float()
        if a2 is not None:
            A = torch.cat([A, a2.float()], 1)
        if m is not None:
            A = A[:m]
        y = A @ W.t()
    rows = y.shape[0]
    if bias is not None:
        if bias_batch_stride:
            assert bias.dim() == 2 and bias.shape[1] == n and rows_per_batch > 0
            y = (y.reshape(rows // rows_per_batch, rows_per_batch, n) + bias[:, None, :]).reshape(rows, n)
        else:
            y = y + bias.reshape(1, n)
    if residual is not None:
        y = y + residual.float()
    return _h(y)


def two_source_attention(q, k0, vt0, n0, **kw):
    return fake_ops.attention(q, k0, vt0, n0, **kw)


def group_norm(x1, gamma, beta, *, batch, hw, eps, silu, x2=None):
    return fake_ops.groupnorm(x1, gamma, beta, batch=batch, hw=hw, eps=eps, silu=silu, x2=x2)


def layer_norm(x, gamma, beta, *, eps=1e-5):
    return fake_ops.layernorm(x, gamma, beta, eps)


def geglu(h):
    """h = [value | gate] in ff.net.0.proj's own row order"""
    n = h.shape[1] // 2
    return _h(h[:, :n].float() * F.gelu(h[:, n:].float()))


def direct_conv3x3(x, wt, *, batch, h, w, cin, cout, stride=1, silu=False, w_param=None, bias=None, residual=None):
    assert x.dtype == torch.float16 and tuple(x.shape) == (batch * h * w, cin) and tuple(wt.shape) == (cout, 9 * cin)
    W = _weight(wt, w_param) if w_param is not None else _unpack(wt, (cout, cin, 3, 3))
    y = F.conv2d(x.float().reshape(batch, h, w, cin).permute(0, 3, 1, 2), W, bias, padding=1, stride=stride)
    if silu:
        y = F.silu(y)
    y = y.permute(0, 2, 3, 1).reshape(-1, cout)
    if residual is not None:
        y = y + residual.float()
    return _h(y)


def skinny_linear_ad(x, w, bias=None, *, w_param=None, silu_in=False):
    assert x.dtype == torch.float32
    W = _weight(w, w_param) if w_param is not None else w.float()
    y = (F.silu(x) if silu_in else x) @ W.t()
    return y if bias is None else y + bias


def upsample_2x(x, *, batch, h, w, c):
    return fake_ops.upsample2x(x, batch=batch, h=h, w=w, c=c)


def add_ad(a, b, *, batch):
    assert a.shape == b.shape
    return _h(a.float() + b.float())


def nchw_to_nhwc(x):
    return fake_ops.nchw_f32_to_nhwc_f16(x)


def nhwc_to_nchw(x, *, batch, c, h, w):
    return fake_ops.nhwc_f16_to_nchw_f32(x, batch=batch, c=c, h=h, w=w)


timestep_embedding = fake_ops.timestep_embedding
ensure_device = fake_ops.ensure_device
require_cuda = fake_ops.require_cuda
