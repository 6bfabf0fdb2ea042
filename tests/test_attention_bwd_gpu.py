"""Attention backward on the GPU: per-shape gradient numerics (tests/attention_bwd_cases.py), determinism, the
LSE-storing forward, and the autograd wrapper."""
import pytest
import torch

from tests import attention_bwd_cases as A
from tests import kernel_cases as K

pytestmark = pytest.mark.gpu

SHAPES = [  # (batch, heads, d, nq, n0, n1, bank_batches, ldv_pad)
    (2, 8, 40, 1024, 1024, 1024, 1, False),
    (2, 8, 80, 200, 77, 0, None, True),
    (2, 8, 160, 256, 256, 64, None, False),
]


@pytest.mark.parametrize("args", A.CASES, ids=[A.case_id(a) for a in A.CASES])
def test_backward_matches_torch_fp32(args):
    err, tol, desc = A.run_case(args)
    torch.cuda.synchronize()
    print(desc)
    assert err <= tol, f"{desc}: error {err:.3e} > {tol:.1e}"


def _setup(batch, heads, d, nq, n0, n1, bank_batches, ldv_pad):
    from magicdance_b200 import ops
    q, k0, v0, vt0, ldv, k1, v1, dout = A.attention_bwd_inputs(batch, heads, d, nq, n0, n1, ldv_pad, seed=7)
    kw = dict(heads=heads, d=d, batch=batch, nq=nq, ldv0_batch=ldv)
    if n1:
        kw.update(k1=k1, vt1=v1.t().contiguous(), n1=n1, kv1_batches=batch,
                  bank_batches=batch if bank_batches is None else bank_batches)
    lse = torch.empty(batch, heads, nq, dtype=torch.float32, device="cuda")
    out = ops.attention(q, k0, vt0, n0, lse=lse, **kw)
    return ops, q, k0, v0, vt0, ldv, k1, v1, dout, kw, lse, out


@pytest.mark.parametrize("shape", SHAPES)
def test_backward_is_bit_reproducible(shape):
    ops, q, k0, v0, vt0, ldv, k1, v1, dout, kw, lse, out = _setup(*shape)
    g1 = ops.attention_backward(q, k0, vt0, shape[4], out, dout, lse, **kw)
    g2 = ops.attention_backward(q, k0, vt0, shape[4], out, dout, lse, **kw)
    torch.cuda.synchronize()
    for a, b in zip(g1, g2):
        assert (a is None and b is None) or torch.equal(a, b)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("two_per_sm", [False, True])
def test_lse_forward_output_is_bit_equal_and_lse_matches_torch(shape, two_per_sm):
    """the LSE-storing forward computes `out` exactly as mdb_attention_f16 does (at d = 40 also on the two-CTA-per-SM
    variant), and its LSE is torch.logsumexp of the scaled fp32 scores"""
    batch, heads, d, nq, n0, n1, bank_batches, _ = shape
    with K.ops.tuning(attn40_2q_min_ctas=0 if two_per_sm else 1 << 30):
        ops, q, k0, v0, vt0, ldv, k1, v1, dout, kw, lse, out = _setup(*shape)
        plain = ops.attention(q, k0, vt0, n0, **kw)
        torch.cuda.synchronize()
    assert torch.equal(out, plain)
    bb = batch if bank_batches is None else bank_batches
    ref = []
    for b in range(batch):
        qq = q[b * nq:(b + 1) * nq].float().reshape(nq, heads, d).transpose(0, 1)
        kk = k0[b * n0:(b + 1) * n0].float()
        if n1 and b < bb:
            kk = torch.cat([kk, k1[b * n1:(b + 1) * n1].float()], 0)
        kk = kk.reshape(-1, heads, d).transpose(0, 1)
        ref.append(torch.logsumexp((qq @ kk.transpose(1, 2)) * d ** -0.5, -1))
    err = float((lse - torch.stack(ref)).abs().max())
    assert err <= 1e-4, err


@pytest.mark.parametrize("shape", SHAPES)
def test_autograd_function_matches_torch_fp32(shape):
    """a scalar loss through ops.two_source_attention (TwoSourceAttention) against torch fp32 autograd of the
    reference formula on the same fp16 inputs"""
    with torch.enable_grad():  # other tests switch autograd off process-wide
        _autograd_vs_torch(shape)


def _autograd_vs_torch(shape):
    from magicdance_b200 import ops
    batch, heads, d, nq, n0, n1, bank_batches, ldv_pad = shape
    bb = batch if bank_batches is None else bank_batches
    q, k0, v0, vt0, ldv, k1, v1, dout = A.attention_bwd_inputs(batch, heads, d, nq, n0, n1, ldv_pad, seed=11)
    w = dout.float()
    leaves = [q.clone(), k0.clone(), vt0.clone()] + ([k1.clone(), v1.t().contiguous()] if n1 else [])
    for t in leaves:
        t.requires_grad_()
    kw = dict(heads=heads, d=d, batch=batch, nq=nq, ldv0_batch=ldv)
    if n1:
        kw.update(k1=leaves[3], vt1=leaves[4], n1=n1, kv1_batches=batch, bank_batches=bb)
    out = ops.two_source_attention(leaves[0], leaves[1], leaves[2], n0, **kw)
    (out.float() * w).sum().backward()

    qf, k0f, v0f = (t.float().requires_grad_() for t in (q, k0, v0))
    k1f, v1f = (k1.float().requires_grad_(), v1.float().requires_grad_()) if n1 else (None, None)
    ref = A.attention_reference(qf, k0f, v0f, k1f, v1f, batch=batch, heads=heads, d=d, nq=nq, n0=n0, n1=n1,
                                bank_batches=bb)
    (ref * w).sum().backward()
    errs = [K.rel(leaves[0].grad.float(), qf.grad), K.rel(leaves[1].grad.float(), k0f.grad),
            K.rel(A.vt_to_tokens(leaves[2].grad, n0, ldv, batch).float(), v0f.grad)]
    if n1:
        errs += [K.rel(leaves[3].grad.float(), k1f.grad), K.rel(A.vt_to_tokens(leaves[4].grad, n1, n1, batch).float(),
                                                                  v1f.grad)]
    assert max(errs) <= 5e-3, errs


def test_shared_source_is_rejected():
    from magicdance_b200 import ops
    ops, q, k0, v0, vt0, ldv, k1, v1, dout, kw, lse, out = _setup(2, 8, 40, 128, 128, 64, None, False)
    kw.update(kv1_batches=1, k1=k1[:64], vt1=v1[:64].t().contiguous())
    with pytest.raises(RuntimeError, match="shared source 1"):
        ops.attention_backward(q, k0, vt0, 128, out, dout, lse, **kw)
