"""TEST DOUBLES — CPU stand-ins for ops.conv3x3_igemm (inference) and ops.conv3x3_igemm_ad (training), the 3x3 conv at
latent sizes that do not tile into the box path's TMA boxes.  They read the kernels' layouts (NHWC fp16 [B*H*W, C]
activations, an optional second source for the upper channels, [O][kh][kw][I] weights), check them, round the output
to fp16, and (training) take the weight term from the fp32 parameter beside its fp16 copy like
tests/fake_train_ops.py.  Every call is counted per (h, w), so a test can see that the path was taken.  Never imported
by the product."""
import collections

import torch
import torch.nn.functional as F

from tests import fake_train_ops

CALLS = collections.Counter()


def _conv(x, w_oihw, x2, conv, conv_stride, bias, bias_batch_stride, rows_per_batch, residual):
    nb, h, wd, c = conv
    assert conv_stride in (1, 2) and x.dtype == torch.float16 and x.dim() == 2 and x.shape[0] == nb * h * wd
    assert x.shape[1] + (0 if x2 is None else x2.shape[1]) == c and w_oihw.shape[1] == c
    if x2 is not None:
        assert x2.dtype == torch.float16 and x.shape[1] % 64 == 0
    CALLS[(h, wd)] += 1
    xs = x.float() if x2 is None else torch.cat([x.float(), x2.float()], 1)
    y = F.conv2d(xs.reshape(nb, h, wd, c).permute(0, 3, 1, 2), w_oihw, None, padding=1, stride=conv_stride)
    n = w_oihw.shape[0]
    y = y.permute(0, 2, 3, 1).reshape(-1, n)
    if bias is not None:
        if bias_batch_stride:
            assert bias.dim() == 2 and bias.shape[1] == n and y.shape[0] == bias.shape[0] * rows_per_batch
            y = (y.reshape(-1, rows_per_batch, n) + bias[:, None, :]).reshape(-1, n)
        else:
            y = y + bias.reshape(1, n)
    if residual is not None:
        y = y + residual.float()
    return y.to(torch.float16)


def conv3x3_igemm(x, w, *, conv, conv_stride=1, x2=None, out=None, bias=None, bias_batch_stride=0, rows_per_batch=0,
                  residual=None, splits=0):
    n, k = w.shape
    c = conv[3]
    assert w.dtype == torch.float16 and k == 9 * c
    y = _conv(x, w.float().reshape(n, 3, 3, c).permute(0, 3, 1, 2), x2, conv, conv_stride, bias, bias_batch_stride,
              rows_per_batch, residual)
    if out is not None:
        out[:y.shape[0]].copy_(y)
        return out
    return y


def conv3x3_igemm_ad(x, w, *, w_param=None, bias=None, bias_batch_stride=0, rows_per_batch=0, residual=None, x2=None,
                     conv, conv_stride=1, splits=0):
    n, k = w.shape
    c = conv[3]
    assert w.dtype == torch.float16 and k == 9 * c
    W = fake_train_ops._weight(w, w_param) if w_param is not None else w.float().reshape(n, 3, 3, c).permute(0, 3, 1, 2)
    return _conv(x, W, x2, conv, conv_stride, bias, bias_batch_stride, rows_per_batch, residual)
