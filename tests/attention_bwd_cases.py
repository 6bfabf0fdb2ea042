"""Numerics cases of the attention backward (ops.attention_backward): each case runs the LSE-storing forward and the
backward on the GPU and returns (error, tolerance, description) against torch float64 autograd of the reference
formula computed from the SAME fp16-rounded inputs.  Run by tests/test_attention_bwd_gpu.py; the same (error,
tolerance, description) contract as tests/kernel_cases.py.

Every output (out, lse, dq, dk*, dvt*) goes into a NaN-poisoned, guarded buffer (tests/kernel_guard.py), so an element
that is never written, or a write outside the output, fails the case.  The padding columns of dvt* and the bank rows
(dk1) and columns (dvt1) of samples >= bank_batches must keep the sentinel: the kernels do not write them.  The
row-stride padding of q, k*, dout and out holds NaN, the "attn_bwd" workspace holds NaN before each call, the
backward runs twice and must be bit-equal, and dq, dk and dv are gated per block of 64 tokens x one head of one
sample, as the forward is."""
import torch

from magicdance_b200 import _lib, ops
from tests.kernel_cases import DEV, _rand, nan_padded
from tests.kernel_guard import Guarded, bit_equal, check_workspace_used, gated, poison_workspace

TOL = 5e-3


def attention_bwd_inputs(batch, heads, d, nq, n0, n1=0, ldv_pad=False, seed=0, pad=0.0):
    """fp16 operands of a two-source attention in the kernel layouts (vt* transposed, per-batch column blocks of
    ldv columns whose padding columns hold `pad`), one bank per batch element; also returns V in token-major layout
    and a gradient of the output."""
    c = heads * d
    q = _rand(batch * nq, c, seed=seed).half()
    k0 = _rand(batch * n0, c, seed=seed + 1).half()
    v0 = _rand(batch * n0, c, seed=seed + 2).half()
    ldv = (n0 + 7) // 8 * 8 if ldv_pad else n0
    vt0 = _vt_cols(v0, n0, ldv, batch, pad)
    k1 = _rand(batch * n1, c, seed=seed + 3).half() if n1 else None
    v1 = _rand(batch * n1, c, seed=seed + 4).half() if n1 else None
    dout = _rand(batch * nq, c, seed=seed + 5).half()
    return q, k0, v0, vt0, ldv, k1, v1, dout


def _vt_cols(v, n, ldv, batch, pad):
    """V [batch*n, c] -> V^T [c, batch*ldv], padding columns holding `pad`"""
    vt = torch.full((v.shape[1], batch * ldv), pad, dtype=torch.float16, device=DEV)
    for b in range(batch):
        vt[:, b * ldv:b * ldv + n] = v[b * n:(b + 1) * n].t()
    return vt


def attention_reference(q, k0, v0, k1, v1, *, batch, heads, d, nq, n0, n1, bank_batches, scale=None):
    """softmax(q k^T scale) v over [self ; bank] per batch element (attention.py:176-198, 303-307), in the inputs'
    dtype; scale defaults to d^-1/2"""
    c = heads * d
    sc = d ** -0.5 if scale is None else scale
    outs = []
    for b in range(batch):
        qq = q[b * nq:(b + 1) * nq].reshape(nq, heads, d).transpose(0, 1)
        kk, vv = k0[b * n0:(b + 1) * n0], v0[b * n0:(b + 1) * n0]
        if n1 and b < bank_batches:
            kk = torch.cat([kk, k1[b * n1:(b + 1) * n1]], 0)
            vv = torch.cat([vv, v1[b * n1:(b + 1) * n1]], 0)
        kk = kk.reshape(-1, heads, d).transpose(0, 1)
        vv = vv.reshape(-1, heads, d).transpose(0, 1)
        s = (qq @ kk.transpose(1, 2)) * sc
        outs.append((s.softmax(-1) @ vv).transpose(0, 1).reshape(nq, c))
    return torch.cat(outs, 0)


def vt_to_tokens(vt, n, ldv, batch):
    """[heads*d][batch*ldv] -> [batch*n][heads*d] (drops the padding columns)"""
    return torch.cat([vt[:, b * ldv:b * ldv + n].t() for b in range(batch)], 0)


def _vt_keep(c, n, ldv, batch, first_unused):
    """the dvt elements the backward must not write: padding columns n..ldv of every sample, and every column of the
    samples >= first_unused"""
    keep = torch.zeros(c, batch * ldv, dtype=torch.bool)
    for b in range(batch):
        keep[:, b * ldv + n:(b + 1) * ldv] = True
    keep[:, first_unused * ldv:] = True
    return keep


def case_attention_bwd(batch, heads, d, nq, n0, n1=0, bank_batches=None, ldv_pad=False, seed=0, pad=0.0, scale=None,
                       sharp=False, bank_pad=None):
    """dq, dk0, dv0, dk1, dv1 against torch float64 autograd; the error is the largest gated rel-L2 of the five.
    pad: the value of vt0's padding columns, which must not reach any gradient; scale: None = d^-1/2; sharp: every
    query is 10 d^-1/2 x one key + 0.5 x itself (its logit against that key is near 10 at every d, a near one-hot
    softmax: 1.6 x the key at d = 40, the forward's case); bank_pad: the value of the bank
    rows of k1 and columns of vt1 of samples >= bank_batches, which nothing may read."""
    bb = batch if bank_batches is None else bank_batches
    c = heads * d
    q, k0, v0, vt0, ldv, k1, v1, dout = attention_bwd_inputs(batch, heads, d, nq, n0, n1, ldv_pad, seed, pad)
    ldv1 = (n1 + 7) // 8 * 8
    if n1:
        vt1 = _vt_cols(v1, n1, ldv1, batch, pad)
        if bank_pad is not None:
            k1[bb * n1:] = bank_pad
            vt1[:, bb * ldv1:] = bank_pad
    if sharp:
        for b in range(batch):
            for i in range(nq):
                tgt = k1[b * n1 + i % n1] if i % 2 and n1 and b < bb else k0[b * n0 + i % n0]
                q[b * nq + i] = (10 * d ** -0.5 * tgt.float() + 0.5 * q[b * nq + i].float()).half()
    q, k0, dout = nan_padded(q), nan_padded(k0), nan_padded(dout)
    kw = dict(heads=heads, d=d, batch=batch, nq=nq, ldv0_batch=ldv, scale=scale)
    if n1:
        k1 = nan_padded(k1)
        kw.update(k1=k1, vt1=vt1, n1=n1, kv1_batches=batch, ldv1_batch=ldv1, bank_batches=bb)
    desc = (f"attention backward B={batch} h={heads} d={d} nq={nq} n0={n0} n1={n1} bank_b={bb} ldv={ldv} pad={pad} "
            f"scale={scale} sharp={sharp} bank_pad={bank_pad}")
    o = Guarded(batch * nq, c)
    lg = Guarded(batch * heads, nq, torch.float32, contiguous=True, shape=(batch, heads, nq))
    out = ops.attention(q, k0, vt0, n0, out=o.out, lse=lg.out, **kw)
    o.check(desc + " out")
    lg.check(desc + " lse")

    def run(what):
        g = {"q": Guarded(batch * nq, c), "k0": Guarded(batch * n0, c),
             "vt0": Guarded(c, batch * ldv, keep=_vt_keep(c, n0, ldv, batch, batch))}
        if n1:
            keep = torch.zeros(batch * n1, c, dtype=torch.bool)
            keep[bb * n1:] = True
            g["k1"] = Guarded(batch * n1, c, keep=keep)
            g["vt1"] = Guarded(c, batch * ldv1, keep=_vt_keep(c, n1, ldv1, batch, bb))
        ws = poison_workspace("attn_bwd", int(_lib.load().mdb_attention_bwd_ws_floats(batch, heads, nq)), q.device)
        ops.attention_backward(q, k0, vt0, n0, out, dout, lg.out, **kw, **{f"out_d{nm}": t.out for nm, t in g.items()})
        for nm, t in g.items():
            t.check(f"{desc} d{nm}{what}")
        check_workspace_used("attn_bwd", ws, desc, q.device)
        return {nm: t.out for nm, t in g.items()}

    got, again = run(""), run(" (second run)")
    for nm in got:
        if not bit_equal(got[nm], again[nm]):
            raise AssertionError(f"{desc}: d{nm} differs between two runs")

    qf, k0f, v0f = (t.double().requires_grad_() for t in (q, k0, v0))
    k1f, v1f = (k1.double().requires_grad_(), v1.double().requires_grad_()) if n1 else (None, None)
    with torch.enable_grad():  # other tests switch autograd off process-wide
        ref = attention_reference(qf, k0f, v0f, k1f, v1f, batch=batch, heads=heads, d=d, nq=nq, n0=n0, n1=n1,
                                  bank_batches=bb, scale=scale)
        (ref * dout.double()).sum().backward()
    pairs = {"dq": (got["q"], qf.grad, batch), "dk0": (got["k0"], k0f.grad, batch),
             "dv0": (vt_to_tokens(got["vt0"], n0, ldv, batch), v0f.grad, batch)}
    if n1 and bb:  # the bank gradients of samples >= bank_batches are not written (checked above)
        pairs["dk1"] = (got["k1"][:bb * n1], k1f.grad[:bb * n1], bb)
        pairs["dv1"] = (vt_to_tokens(got["vt1"], n1, ldv1, bb), v1f.grad[:bb * n1], bb)
    errs, notes = {}, ""
    for nm, (g_, r_, groups) in pairs.items():
        errs[nm], note = gated(g_, r_, TOL, rows=64, cols=d, groups=groups)
        notes += f" {nm}{note}"
    return max(errs.values()), TOL, f"{desc}: error " + " ".join(f"{k} {e:.2e}" for k, e in errs.items()) + notes


# (batch, heads, d, nq, n0[, n1, bank_batches, ldv_pad, seed, pad]) or keyword arguments; one bank per sample (shared
# sources are not supported)
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
_NAN = float("nan")
for _d in (40, 80, 160):
    CASES += [
        # one query and one self key (a single key alone makes dq and dk exactly zero, where no relative error
        # means anything, so a bank follows it)
        dict(batch=2, heads=8, d=_d, nq=1, n0=1, n1=100, ldv_pad=True, pad=_NAN),
        dict(batch=1, heads=8, d=_d, nq=1, n0=1, n1=64, ldv_pad=True),
        dict(batch=2, heads=1, d=_d, nq=200, n0=200, n1=64),                          # one head
        dict(batch=2, heads=8, d=_d, nq=300, n0=100, n1=0, ldv_pad=True, pad=_NAN),  # more queries than keys
        dict(batch=2, heads=8, d=_d, nq=100, n0=300, n1=72, ldv_pad=True, pad=_NAN),  # fewer
        dict(batch=2, heads=8, d=_d, nq=60, n0=77, ldv_pad=True, pad=_NAN),          # text K / V at a 40x24 level
        dict(batch=2, heads=8, d=_d, nq=200, n0=200, n1=64, scale=0.3),               # an explicit scale
        dict(batch=2, heads=8, d=_d, nq=256, n0=256, n1=256, sharp=True),            # a near one-hot softmax
        # NaN / Inf in the bank keys and values of the samples without a bank, n1 ragged: the last bank key tile of
        # sample bank_batches - 1 must not reach into them
        dict(batch=2, heads=8, d=_d, nq=200, n0=200, n1=100, bank_batches=1, bank_pad=_NAN),
        dict(batch=3, heads=8, d=_d, nq=130, n0=136, n1=36, bank_batches=2, ldv_pad=True, pad=_NAN,
             bank_pad=float("inf")),
    ]
CASES += [
    # the self + bank attention of a 40x24 latent at batch 2 (15 / 60 / 240 / 960 tokens per level)
    dict(batch=2, heads=8, d=160, nq=15, n0=15, n1=15, ldv_pad=True, pad=_NAN),
    dict(batch=2, heads=8, d=160, nq=60, n0=60, n1=60, ldv_pad=True, pad=_NAN),
    dict(batch=2, heads=8, d=80, nq=240, n0=240, n1=240),
    dict(batch=2, heads=8, d=40, nq=960, n0=960, n1=960),
    dict(batch=2, heads=8, d=40, nq=960, n0=77, ldv_pad=True, pad=_NAN),
]


def case_id(args):
    if isinstance(args, dict):
        return "-".join(f"{k}={v}" for k, v in args.items())
    return "-".join(map(str, args))


def run_case(args):
    return case_attention_bwd(**args) if isinstance(args, dict) else case_attention_bwd(*args)
