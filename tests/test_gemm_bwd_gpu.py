"""GEMM / convolution backward on the GPU: per-shape gradient numerics (tests/gemm_bwd_cases.py), bit-reproducibility
of the split reductions, the autograd op on a small conv -> SiLU -> stride-2 conv -> Linear chain, and one attention
layer whose projections and attention both run backward through library kernels."""
import pytest
import torch
import torch.nn.functional as F

from tests import attention_bwd_cases as A
from tests import gemm_bwd_cases as G
from tests.kernel_cases import _rand, rel

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kw", G.CASES, ids=[G.case_id(c) for c in G.CASES])
def test_backward_matches_torch_fp32(kw):
    err, tol, desc = G.case_gemm_bwd(**kw)
    torch.cuda.synchronize()
    print(desc)
    assert err <= tol, f"{desc}: error {err:.3e} > {tol:.1e}"


@pytest.mark.parametrize("conv", [None, (2, 32, 32)])
def test_backward_is_bit_reproducible(conv):
    """every output of a call whose reductions are split (fp32 slabs summed in a fixed order) is bit-equal run to run"""
    from magicdance_b200 import ops
    if conv is None:
        a, w = _rand(2048, 640, seed=1).half(), _rand(640, 640, seed=2, scale=0.04).half()
        kw = dict(splits=4, db_splits=6)
        m = 2048
    else:
        a, w = _rand(2 * 32 * 32, 320, seed=1).half(), _rand(320, 9 * 320, seed=2, scale=0.02).half()
        kw = dict(conv=(2, 32, 32, 320), splits=3, db_splits=4)
        m = 2 * 32 * 32
    dd = _rand(m, w.shape[0], seed=3).half()
    kw.update(grads=("a", "b", "bias"))
    g1 = ops.gemm_backward(a, w, dd, **kw)
    g2 = ops.gemm_backward(a, w, dd, **kw)
    torch.cuda.synchronize()
    for x, y in zip(g1, g2):
        assert (x is None and y is None) or torch.equal(x, y)


def test_autograd_chain_matches_torch_fp32():
    """conv3x3 -> torch SiLU -> stride-2 conv3x3 -> Linear with a per-batch bias through ops.tc_gemm, against
    F.conv2d / F.linear autograd in fp32 on the same fp16-rounded parameters: the input gradient and every
    parameter gradient"""
    with torch.enable_grad():  # other tests switch autograd off process-wide
        _chain()


def _chain():
    from magicdance_b200 import ops
    nb, h, w, c0, c1, c2, c3 = 2, 16, 16, 64, 64, 128, 64
    x = _rand(nb, c0, h, w, seed=1).half().float()
    w1 = _rand(c1, c0, 3, 3, seed=2, scale=(9 * c0) ** -0.5).half().float()
    w2 = _rand(c2, c1, 3, 3, seed=3, scale=(9 * c1) ** -0.5).half().float()
    w3 = _rand(c3, c2, seed=4, scale=c2 ** -0.5).half().float()
    b3 = _rand(nb, c3, seed=5).float()
    g = _rand(nb, (h // 2) * (w // 2), c3, seed=6)
    pack = lambda p: p.permute(0, 2, 3, 1).reshape(p.shape[0], -1).half().contiguous()  # OIHW -> [O][kh][kw][I]
    params = [t.clone().requires_grad_() for t in (w1, w2, w3, b3)]
    xh = x.permute(0, 2, 3, 1).reshape(-1, c0).half().contiguous().requires_grad_()
    y1 = ops.tc_gemm(xh, pack(params[0]), w_param=params[0], conv=(nb, h, w, c0))
    y1 = F.silu(y1)
    y2 = ops.tc_gemm(y1, pack(params[1]), w_param=params[1], conv=(nb, h, w, c1), conv_stride=2)
    y3 = ops.tc_gemm(y2, params[2].half(), w_param=params[2], bias=params[3], bias_batch_stride=c3,
                     rows_per_batch=(h // 2) * (w // 2))
    (y3.float() * g.reshape(-1, c3)).sum().backward()

    refs = [t.clone().requires_grad_() for t in (x, w1, w2, w3, b3)]
    r = F.silu(F.conv2d(refs[0], refs[1], padding=1))
    r = F.conv2d(r, refs[2], stride=2, padding=1).permute(0, 2, 3, 1).reshape(nb, -1, c2)
    r = F.linear(r, refs[3]) + refs[4][:, None, :]
    (r * g).sum().backward()
    errs = {"dx": rel(xh.grad.float(), refs[0].grad.permute(0, 2, 3, 1).reshape(-1, c0))}
    for nm, p, ref in zip(("dw1", "dw2", "dw3", "db3"), params, refs[1:]):
        assert p.grad.shape == ref.grad.shape and p.grad.dtype == torch.float32, nm
        errs[nm] = rel(p.grad, ref.grad)
    print(errs)
    assert max(errs.values()) <= 1e-2, errs


def test_attention_layer_backward_through_library_kernels():
    """self tokens x and bank tokens x_bank -> q / k by gemm(., W), V^T by gemm(Wv, .) -> ops.two_source_attention ->
    scalar loss: dx, dx_bank, dWq, dWk, dWv against torch fp32 autograd.  Wk and Wv are each used twice, so autograd
    sums two fp32 contributions into their gradients."""
    with torch.enable_grad():
        _attention_layer()


def _attention_layer():
    from magicdance_b200 import ops
    heads, d, n0, n1 = 8, 40, 256, 256
    c = heads * d
    x = _rand(n0, c, seed=1).half()
    xb = _rand(n1, c, seed=2).half()
    ws = [_rand(c, c, seed=3 + i, scale=c ** -0.5).half().float() for i in range(3)]
    g = _rand(n0, c, seed=9)
    params = [t.clone().requires_grad_() for t in ws]
    xs = [t.clone().requires_grad_() for t in (x, xb)]
    wq, wk, wv = params
    q = ops.tc_gemm(xs[0], wq.half(), w_param=wq)
    k0 = ops.tc_gemm(xs[0], wk.half(), w_param=wk)
    k1 = ops.tc_gemm(xs[1], wk.half(), w_param=wk)
    vt0 = ops.tc_gemm(wv.half(), xs[0], a_param=wv)
    vt1 = ops.tc_gemm(wv.half(), xs[1], a_param=wv)
    out = ops.two_source_attention(q, k0, vt0, n0, heads=heads, d=d, batch=1, nq=n0, k1=k1, vt1=vt1, n1=n1,
                                   kv1_batches=1, bank_batches=1)
    (out.float() * g).sum().backward()

    rx, rxb = (t.float().requires_grad_() for t in (x, xb))
    rw = [t.clone().requires_grad_() for t in ws]
    ref = A.attention_reference(F.linear(rx, rw[0]), F.linear(rx, rw[1]), F.linear(rx, rw[2]), F.linear(rxb, rw[1]),
                                F.linear(rxb, rw[2]), batch=1, heads=heads, d=d, nq=n0, n0=n0, n1=n1, bank_batches=1)
    (ref * g).sum().backward()
    errs = {"dx": rel(xs[0].grad.float(), rx.grad), "dx_bank": rel(xs[1].grad.float(), rxb.grad)}
    for nm, p, r in zip(("dWq", "dWk", "dWv"), params, rw):
        errs[nm] = rel(p.grad, r.grad)
    print(errs)
    assert max(errs.values()) <= 1e-2, errs
