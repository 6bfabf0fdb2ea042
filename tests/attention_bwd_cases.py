"""Numerics cases of the attention backward (ops.attention_backward): each case runs the LSE-storing forward and the
backward on the GPU and returns (error, tolerance, description) against torch fp32 autograd of the reference formula
computed from the SAME fp16-rounded inputs.  Run by tests/test_attention_bwd_gpu.py; the same (error, tolerance,
description) contract as tests/kernel_cases.py."""
import torch

from magicdance_b200 import ops
from tests.kernel_cases import DEV, _rand, rel


def attention_bwd_inputs(batch, heads, d, nq, n0, n1=0, ldv_pad=False, seed=0, pad=0.0):
    """fp16 operands of a two-source attention in the kernel layouts (vt* transposed, per-batch column blocks of
    ldv columns whose padding columns hold `pad`), one bank per batch element; also returns V in token-major layout
    and a gradient of the output."""
    c = heads * d
    q = _rand(batch * nq, c, seed=seed).half()
    k0 = _rand(batch * n0, c, seed=seed + 1).half()
    v0 = _rand(batch * n0, c, seed=seed + 2).half()
    ldv = (n0 + 7) // 8 * 8 if ldv_pad else n0
    vt0 = torch.full((c, batch * ldv), pad, dtype=torch.float16, device=DEV)
    for b in range(batch):
        vt0[:, b * ldv:b * ldv + n0] = v0[b * n0:(b + 1) * n0].t()
    k1 = _rand(batch * n1, c, seed=seed + 3).half() if n1 else None
    v1 = _rand(batch * n1, c, seed=seed + 4).half() if n1 else None
    dout = _rand(batch * nq, c, seed=seed + 5).half()
    return q, k0, v0, vt0, ldv, k1, v1, dout


def attention_reference(q, k0, v0, k1, v1, *, batch, heads, d, nq, n0, n1, bank_batches):
    """fp32 softmax(q k^T d^-1/2) v over [self ; bank] per batch element (attention.py:176-198, 303-307)"""
    c = heads * d
    outs = []
    for b in range(batch):
        qq = q[b * nq:(b + 1) * nq].reshape(nq, heads, d).transpose(0, 1)
        kk, vv = k0[b * n0:(b + 1) * n0], v0[b * n0:(b + 1) * n0]
        if n1 and b < bank_batches:
            kk = torch.cat([kk, k1[b * n1:(b + 1) * n1]], 0)
            vv = torch.cat([vv, v1[b * n1:(b + 1) * n1]], 0)
        kk = kk.reshape(-1, heads, d).transpose(0, 1)
        vv = vv.reshape(-1, heads, d).transpose(0, 1)
        s = (qq @ kk.transpose(1, 2)) * d ** -0.5
        outs.append((s.softmax(-1) @ vv).transpose(0, 1).reshape(nq, c))
    return torch.cat(outs, 0)


def vt_to_tokens(vt, n, ldv, batch):
    """[heads*d][batch*ldv] -> [batch*n][heads*d] (drops the padding columns)"""
    return torch.cat([vt[:, b * ldv:b * ldv + n].t() for b in range(batch)], 0)


def case_attention_bwd(batch, heads, d, nq, n0, n1=0, bank_batches=None, ldv_pad=False, seed=0, pad=0.0):
    """dq, dk0, dv0, dk1, dv1 against torch fp32 autograd; the error is the largest rel-L2 of the five.  Padding
    columns of dvt0 must stay zero; pad: the value of vt0's padding columns, which must not reach any gradient."""
    bb = batch if bank_batches is None else bank_batches
    q, k0, v0, vt0, ldv, k1, v1, dout = attention_bwd_inputs(batch, heads, d, nq, n0, n1, ldv_pad, seed, pad)
    kw = dict(heads=heads, d=d, batch=batch, nq=nq, ldv0_batch=ldv)
    if n1:
        kw.update(k1=k1, vt1=v1.t().contiguous(), n1=n1, kv1_batches=batch, bank_batches=bb)
    lse = torch.empty(batch, heads, nq, dtype=torch.float32, device=DEV)
    out = ops.attention(q, k0, vt0, n0, lse=lse, **kw)
    dq, dk0, dvt0, dk1, dvt1 = ops.attention_backward(q, k0, vt0, n0, out, dout, lse, **kw)
    qf, k0f, v0f = (t.float().requires_grad_() for t in (q, k0, v0))
    k1f, v1f = (k1.float().requires_grad_(), v1.float().requires_grad_()) if n1 else (None, None)
    with torch.enable_grad():  # other tests switch autograd off process-wide
        ref = attention_reference(qf, k0f, v0f, k1f, v1f, batch=batch, heads=heads, d=d, nq=nq, n0=n0, n1=n1,
                                  bank_batches=bb)
        (ref * dout.float()).sum().backward()
    errs = [rel(dq.float(), qf.grad), rel(dk0.float(), k0f.grad), rel(vt_to_tokens(dvt0, n0, ldv, batch).float(), v0f.grad)]
    if n1:
        errs += [rel(dk1.float(), k1f.grad), rel(vt_to_tokens(dvt1, n1, n1, batch).float(), v1f.grad)]
    pad = sum(float(dvt0[:, b * ldv + n0:(b + 1) * ldv].abs().sum()) for b in range(batch))
    return max(errs) + pad, 5e-3, (f"attention backward B={batch} h={heads} d={d} nq={nq} n0={n0} n1={n1} bank_b={bb} "
                                   f"ldv={ldv}: rel-L2 dq/dk0/dv0/dk1/dv1 " + " ".join(f"{e:.2e}" for e in errs))


# (batch, heads, d, nq, n0[, n1, bank_batches, ldv_pad, seed, pad]); one bank per sample (shared sources are not
# supported)
CASES = [
    (1, 8, 40, 4096, 4096, 4096),      # self + bank at 64x64
    (2, 8, 40, 1024, 1024, 1024),
    (2, 8, 40, 1024, 1024, 1024, 1),   # bank_batches < batch: the second sample has no bank
    (2, 8, 40, 1024, 77, 0, None, True),   # 77 text tokens, ldv padded to 80
    (1, 8, 40, 384, 384, 128),         # n1 = 128 against n0 = 384, odd number of Q tiles
    (2, 8, 80, 256, 256, 256),
    (2, 8, 80, 200, 200, 0),           # ragged nq and n0
    (2, 8, 80, 1024, 77, 0, None, True),
    (1, 8, 160, 320, 320, 64),
    (2, 8, 160, 64, 64, 64),
    (1, 8, 160, 16, 16, 16),
    (2, 8, 160, 256, 77, 0, None, True),
    (2, 8, 160, 200, 200, 200, 1),     # ragged, and bank_batches < batch
    # NaN in vt0's padding columns: the dQ kernel's dP = dO V^T must not read them
    (2, 8, 40, 1024, 77, 0, None, True, 0, float("nan")),
    (2, 8, 80, 63, 63, 0, None, True, 0, float("nan")),            # nq and n0 below one 64-row step
    (2, 8, 40, 50, 33, 24, None, True, 0, float("nan")),
    (1, 8, 160, 33, 40, 16, None, True, 0, float("nan")),
]
