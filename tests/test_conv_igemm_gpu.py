"""The 3x3 convolution at any latent size on the GPU (ops.conv3x3_igemm / conv3x3_igemm_backward / conv3x3_igemm_ad):
forward and gradient numerics against torch fp32 (tests/igemm_cases.py), bit-equality with the box path at the sizes
both take, bit-reproducible backward, and the autograd op."""
import pytest
import torch
import torch.nn.functional as F

from tests import igemm_cases as I
from tests.kernel_cases import _rand, rel

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kw", I.FWD_CASES, ids=[I.case_id(c) for c in I.FWD_CASES])
def test_forward_matches_torch_fp32(kw):
    err, tol, desc = I.case_fwd(**kw)
    torch.cuda.synchronize()
    print(desc)
    assert err <= tol, f"{desc}: error {err:.3e} > {tol:.1e}"


@pytest.mark.parametrize("kw", I.BWD_CASES, ids=[I.case_id(c) for c in I.BWD_CASES])
def test_backward_matches_torch_fp32(kw):
    err, tol, desc = I.case_bwd(**kw)
    torch.cuda.synchronize()
    print(desc)
    assert err <= tol, f"{desc}: error {err:.3e} > {tol:.1e}"


@pytest.mark.parametrize("nb,h,w,cin,cout,stride", [
    (2, 64, 64, 320, 320, 1), (1, 64, 64, 320, 320, 2), (2, 32, 32, 640, 640, 1), (2, 32, 32, 640, 640, 2),
    (4, 16, 16, 1280, 1280, 1), (2, 8, 8, 1280, 1280, 1), (2, 64, 64, 960, 320, 1)])
def test_bit_equal_to_the_box_path(nb, h, w, cin, cout, stride):
    """where the pixels tile into TMA boxes, the im2col loads give the same tiles: forward and every gradient agree to
    the bit"""
    (y_box, y_im), grads = I.box_vs_im2col(nb, h, w, cin, cout, stride)
    torch.cuda.synchronize()
    assert torch.equal(y_box, y_im), f"forward differs: max {float((y_box.float() - y_im.float()).abs().max()):.3e}"
    for i, (p, q) in enumerate(grads):
        assert torch.equal(p, q), f"gradient {i} differs: max {float((p.float() - q.float()).abs().max()):.3e}"


def test_backward_is_bit_reproducible():
    from magicdance_b200 import ops
    x, x2 = _rand(2 * 14 * 8, 640, seed=1).half(), _rand(2 * 14 * 8, 640, seed=4).half()
    w = _rand(640, 9 * 1280, seed=2, scale=0.01).half()
    dd = _rand(2 * 14 * 8, 640, seed=3).half()
    kw = dict(conv=(2, 14, 8, 1280), x2=x2, splits=3, db_splits=4, grads=("a", "b", "bias"))
    g1 = ops.conv3x3_igemm_backward(x, w, dd, **kw)
    g2 = ops.conv3x3_igemm_backward(x, w, dd, **kw)
    torch.cuda.synchronize()
    for p, q in zip(g1, g2):
        assert torch.equal(p, q)


def test_autograd_op_matches_torch():
    """conv3x3_igemm_ad with an fp32 OIHW parameter, a per-image bias and a residual: the gradients reach x, the
    parameter (in its own layout), the bias and the residual"""
    from magicdance_b200 import ops
    nb, h, w, c = 2, 20, 12, 320
    x = _rand(nb * h * w, c, seed=1).half().requires_grad_()
    wp = _rand(c, c, 3, 3, seed=2, scale=0.02).requires_grad_()
    w16 = wp.detach().permute(0, 2, 3, 1).reshape(c, 9 * c).half()
    bias = _rand(nb, c, seed=3).requires_grad_()
    res = _rand(nb * h * w, c, seed=4).half().requires_grad_()
    y = ops.conv3x3_igemm_ad(x, w16, w_param=wp, bias=bias, bias_batch_stride=c, rows_per_batch=h * w, residual=res,
                             conv=(nb, h, w, c))
    dy = _rand(nb * h * w, c, seed=5).half()
    y.backward(dy)
    xr = x.detach().float().reshape(nb, h, w, c).permute(0, 3, 1, 2).requires_grad_()
    wr = w16.float().reshape(c, 3, 3, c).permute(0, 3, 1, 2).detach().requires_grad_()
    br = bias.detach().clone().requires_grad_()
    yr = F.conv2d(xr, wr, padding=1).permute(0, 2, 3, 1).reshape(nb, h * w, c) + br[:, None]
    yr = yr.reshape(-1, c) + res.detach().float()
    yr.backward(dy.float())
    assert rel(y, yr) < 2e-3
    assert rel(x.grad, xr.grad.permute(0, 2, 3, 1).reshape(-1, c)) < 2e-3
    assert wp.grad.shape == wp.shape and rel(wp.grad, wr.grad) < 2e-3
    assert rel(bias.grad, br.grad) < 1e-4
    assert torch.equal(res.grad, dy)
