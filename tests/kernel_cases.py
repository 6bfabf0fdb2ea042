"""Per-kernel numerics cases: each function runs one C-ABI kernel on the GPU and returns
(error, tolerance, description) against a plain PyTorch fp32 reference of the same op computed
from the SAME fp16-rounded inputs.  Shared by tests/test_kernels_gpu.py and scripts/gpu_diag.py.

Every output goes into a NaN-poisoned, guarded buffer or a poisoned allocation (tests/kernel_guard.py): a case
raises AssertionError when an output element was never written or a write landed outside the output.  Operand
padding that a kernel must not read (row-stride padding of A, residual, q and k; the bias columns around a per-batch
bias slice) holds NaN.  GEMM, conv and attention outputs are also gated per block (gated())."""
import math

import torch
import torch.nn.functional as F

from magicdance_b200 import ops
from tests.kernel_guard import Guarded, check_poisoned, gated, poison_, poisoned_alloc, rel  # noqa: F401 (rel: shared)

DEV = "cuda"


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def nan_padded(t, extra=8):
    """t ([rows, cols] fp16) as the column slice of a wider buffer whose other columns hold NaN: a kernel that reads
    past the row's end produces NaN"""
    buf = poison_(torch.empty((t.shape[0], (t.shape[1] + 7) // 8 * 8 + extra), dtype=t.dtype, device=t.device))
    buf[:, :t.shape[1]] = t
    return buf[:, :t.shape[1]]


def guarded_run(rows, cols, launch, desc, twice=False, **kw):
    """launch(out) into a Guarded [rows, cols] buffer (kw: Guarded's options) and check it; with `twice`, launch
    again into a second poisoned buffer and require the two results to be bit-equal (split-K reductions and
    attention promise run-to-run determinism).  Returns the output."""
    o = Guarded(rows, cols, **kw)
    launch(o.out)
    o.check(desc)
    if twice:
        o2 = Guarded(rows, cols, **kw)
        launch(o2.out)
        o2.check(desc + " (second run)")
        if not torch.equal(o.out, o2.out):
            raise AssertionError(f"{desc}: two runs differ")
    return o.out


def case_gemm(m, n, k, bias=False, residual=False, splits=1, seed=0):
    """splits: 0 = the library's choice (possibly split-K in a cluster), n > 1 = exactly n (2 / 4 / 8 reduce in a
    cluster, other counts through the fp32 workspace); every split-K run is repeated and must be bit-equal"""
    a = nan_padded(_rand(m, k, seed=seed).half())
    w = _rand(n, k, seed=seed + 1, scale=k ** -0.5).half()
    b = _rand(n, seed=seed + 2).float() if bias else None
    r = nan_padded(_rand(m, n, seed=seed + 3).half()) if residual else None
    desc = f"gemm m={m} n={n} k={k} bias={bias} res={residual} splits={splits}"
    out = guarded_run(m, n, lambda o: ops.gemm(a, w, bias=b, residual=r, splits=splits, out=o), desc, splits != 1)
    ref = a.float() @ w.float().t()
    if bias:
        ref = ref + b
    if residual:
        ref = ref + r.float()
    err, note = gated(out, ref, 2e-3)
    return err, 2e-3, desc + note


def case_tuned(tune, fn, *args):
    """Runs another case under `ops.tuning(**tune)` — the library's launch heuristics (mdb_set_tuning) — so that a
    kernel variant that the heuristics reserve for large grids is exercised on a small problem.
    tune: tuple of (name, value) pairs, e.g. (("pair_min_tiles", 1),)."""
    with ops.tuning(**dict(tune)):
        err, tol, desc = fn(*args)
        torch.cuda.synchronize()
    return err, tol, " ".join(f"{k}={v}" for k, v in tune) + ": " + desc


PAIR = (("pair_min_tiles", 1),)     # the large-grid tiles (128 x 256 / deep rings, one CTA per SM) whatever the grid size
NOPAIR = (("pair_min_tiles", 1 << 30),)  # the small-grid tiles (two CTAs per SM up to 128 wide) on a large grid
ATT2Q = (("attn40_2q_min_ctas", 0),)     # d=40 attention on the register-capped variant at two CTAs per SM
BN160 = (("bn80_below", 0),)   # N % 160 == 0 on the 160-wide small-grid tiles whatever the grid size


def case_gemm_ln(m, n, k, offset=0.5, seed=0):
    """LayerNorm folded into the GEMM (ops.gemm(ln_u=...), engine.fold_layernorm) against LayerNorm -> Linear in fp32;
    offset: row mean of the activations (the correction rstd (acc - mean u) must not cancel)."""
    from magicdance_b200.engine import fold_layernorm
    x = nan_padded((_rand(m, k, seed=seed) * 1.3 + offset).half())
    w = _rand(n, k, seed=seed + 1, scale=k ** -0.5)
    gamma = 1 + 0.1 * _rand(k, seed=seed + 2)
    beta = 0.1 * _rand(k, seed=seed + 3)
    b = 0.1 * _rand(n, seed=seed + 4)
    w_ln, u, v = fold_layernorm(w, gamma, beta, b, DEV)
    o = Guarded(m, n)
    ops.gemm(x, w_ln, bias=v, ln_u=u, ln_eps=1e-5, out=o.out)
    desc = f"gemm with folded LayerNorm m={m} n={n} k={k} offset={offset}"
    o.check(desc)
    ref = F.layer_norm(x.double(), (k,), gamma.double(), beta.double(), 1e-5) @ w.double().t() + b.double()
    err, note = gated(o.out, ref, 3e-3)
    return err, 3e-3, desc + note


def case_gemm_batch_bias(batch, hw, n, k, splits=0, seed=0):
    """per-sample bias rows (the ResBlock's timestep bias); hw = rows_per_batch: below 128 one tile holds several
    samples.  The bias buffer's columns outside the slice hold NaN."""
    m = batch * hw
    a = _rand(m, k, seed=seed).half()
    w = _rand(n, k, seed=seed + 1, scale=k ** -0.5).half()
    ball = poison_(torch.empty(batch, n + 64, device=DEV))
    bias = ball[:, 32:32 + n]
    bias.copy_(_rand(batch, n, seed=seed + 2))
    desc = f"gemm per-batch bias B={batch} hw={hw} n={n} k={k} splits={splits}"
    out = guarded_run(m, n, lambda o: ops.gemm(a, w, bias=bias, bias_batch_stride=ball.stride(0), rows_per_batch=hw,
                                               splits=splits, out=o), desc, splits != 1)
    ref = ((a.float() @ w.float().t()).reshape(batch, hw, n) + bias[:, None, :]).reshape(m, n)
    err, note = gated(out, ref, 2e-3)
    return err, 2e-3, desc + note


def case_gemm_dual(m, n, k1, k2, splits=1, seed=0):
    """A = [a1 | a2] from two sources; with splits the k1 boundary may fall inside a split"""
    a1 = nan_padded(_rand(m, k1, seed=seed).half())
    a2 = nan_padded(_rand(m, k2, seed=seed + 5).half())
    w = _rand(n, k1 + k2, seed=seed + 1, scale=(k1 + k2) ** -0.5).half()
    desc = f"gemm dual-source m={m} n={n} k={k1}+{k2} splits={splits}"
    out = guarded_run(m, n, lambda o: ops.gemm(a1, w, a2=a2, splits=splits, out=o), desc, splits != 1)
    ref = torch.cat([a1, a2], 1).float() @ w.float().t()
    err, note = gated(out, ref, 2e-3)
    return err, 2e-3, desc + note


def case_gemm_strided_out(m, n, k, seed=0):
    """D written into a column slice of a wider buffer (text V^T layout): guard columns on both sides, row pitch > N"""
    a = _rand(m, k, seed=seed).half()
    w = _rand(n, k, seed=seed + 1, scale=k ** -0.5).half()
    o = Guarded(m, n, left=(n + 7) // 8 * 8)
    ops.gemm(a, w, out=o.out)
    desc = f"gemm strided out m={m} n={n} k={k}"
    o.check(desc)
    err, note = gated(o.out, a.float() @ w.float().t(), 2e-3)
    return err, 2e-3, desc + note


def case_geglu(m, c, seed=0):
    from magicdance_b200.engine import pack_geglu
    x = nan_padded(_rand(m, c, seed=seed).half())
    w = _rand(8 * c, c, seed=seed + 1, scale=c ** -0.5)
    b = _rand(8 * c, seed=seed + 2, scale=0.1)
    wp, bp = pack_geglu(w, b, DEV)
    o = Guarded(m, 4 * c)
    ops.gemm(x, wp, bias=bp, epilogue=ops.EPI_GEGLU, out=o.out)
    desc = f"geglu m={m} c={c}"
    o.check(desc)
    y = x.float() @ w.half().float().t() + b
    v, g = y.chunk(2, dim=-1)
    err, note = gated(o.out, v * F.gelu(g), 3e-3)
    return err, 3e-3, desc + note


def case_conv(batch, h, w, cin, cout, bias=True, residual=False, splits=1, batch_bias=False, seed=0):
    """batch_bias: one bias row per image (the ResBlock's timestep bias, rows_per_batch = h*w)"""
    x = _rand(batch, cin, h, w, seed=seed).half()
    wt = _rand(cout, cin, 3, 3, seed=seed + 1, scale=(9 * cin) ** -0.5).half()
    b = _rand(batch if batch_bias else 1, cout, seed=seed + 2).float() if bias else None
    bkw = dict(bias_batch_stride=cout, rows_per_batch=h * w) if batch_bias else {}
    from magicdance_b200.engine import pack_conv3x3
    xn = x.permute(0, 2, 3, 1).contiguous().reshape(batch * h * w, cin)
    r = nan_padded(_rand(batch * h * w, cout, seed=seed + 3).half()) if residual else None
    wp = pack_conv3x3(wt, DEV)
    desc = f"conv3x3 igemm B={batch} {h}x{w} {cin}->{cout} splits={splits} batch_bias={batch_bias}"
    out = guarded_run(batch * h * w, cout, lambda o: ops.gemm(xn, wp, bias=b, residual=r, conv=(batch, h, w, cin),
                                                              splits=splits, out=o, **bkw), desc, splits != 1)
    ref = F.conv2d(x.float(), wt.float(), padding=1)
    if bias:
        ref = ref + b[:, :, None, None]
    ref = ref.permute(0, 2, 3, 1).reshape(batch * h * w, cout)
    if residual:
        ref = ref + r.float()
    err, note = gated(out, ref, 2e-3)
    return err, 2e-3, desc + note


def case_conv_s2(batch, h, w, cin, cout, seed=0):
    """3x3 stride-2 pad-1 conv (Downsample.op, openaimodel.py:175) as implicit GEMM: TMA element strides of 2"""
    x = _rand(batch * h * w, cin, seed=seed).half()
    wt = _rand(cout, 3, 3, cin, seed=seed + 1, scale=(9 * cin) ** -0.5).half()
    b = _rand(cout, seed=seed + 2).float()
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    o = Guarded(batch * ho * wo, cout)
    ops.gemm(x, wt.reshape(cout, 9 * cin), bias=b, conv=(batch, h, w, cin), conv_stride=2, out=o.out)
    desc = f"conv 3x3 stride 2 (implicit GEMM) B={batch} {h}x{w} {cin}->{cout}"
    o.check(desc)
    xr = x.float().reshape(batch, h, w, cin).permute(0, 3, 1, 2)
    ref = F.conv2d(xr, wt.float().permute(0, 3, 1, 2), b, stride=2, padding=1).permute(0, 2, 3, 1).reshape(-1, cout)
    err, note = gated(o.out, ref, 2e-3)
    return err, 2e-3, desc + note


def case_conv_direct(batch, h, w, cin, cout, stride, silu, residual=False, seed=0):
    x = _rand(batch, cin, h, w, seed=seed).half()
    wt = _rand(cout, cin, 3, 3, seed=seed + 1, scale=(9 * cin) ** -0.5).half()
    b = _rand(cout, seed=seed + 2).float()
    from magicdance_b200.engine import pack_conv3x3
    xn = x.permute(0, 2, 3, 1).contiguous().reshape(batch * h * w, cin)
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    r = _rand(batch * ho * wo, cout, seed=seed + 3).half() if residual else None
    o = Guarded(batch * ho * wo, cout, contiguous=True)
    ops.conv3x3_direct(xn, pack_conv3x3(wt, DEV), b, batch=batch, h=h, w=w, cin=cin, cout=cout, stride=stride,
                       silu=silu, residual=r, out=o.out)
    desc = f"conv3x3 direct B={batch} {h}x{w} {cin}->{cout} s={stride} silu={silu} res={residual}"
    o.check(desc)
    ref = F.conv2d(x.float(), wt.float(), b, padding=1, stride=stride)
    if silu:
        ref = F.silu(ref)
    ref = ref.permute(0, 2, 3, 1).reshape(batch * ho * wo, cout)
    if residual:
        ref = ref + r.float()
    err, note = gated(o.out, ref, 2e-3)
    return err, 2e-3, desc + note


def _im2col(xn, batch, h, w, c, stride, pad):
    """ops.im2col3x3 into a poisoned allocation"""
    if pad == "br":
        ho, wo = (h + 1 - 3) // stride + 1, (w + 1 - 3) // stride + 1
    else:
        ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    ptr = poisoned_alloc((batch * ho * wo, 9 * c), torch.float16)
    col = ops.im2col3x3(xn, batch=batch, h=h, w=w, c=c, stride=stride, pad=pad)
    check_poisoned(col, ptr, f"im2col3x3 B={batch} {h}x{w} c={c} s={stride} pad={pad}")
    return col


def case_down(batch, h, w, c, seed=0):
    x = _rand(batch, c, h, w, seed=seed).half()
    wt = _rand(c, c, 3, 3, seed=seed + 1, scale=(9 * c) ** -0.5).half()
    b = _rand(c, seed=seed + 2).float()
    from magicdance_b200.engine import pack_conv3x3
    xn = x.permute(0, 2, 3, 1).contiguous().reshape(batch * h * w, c)
    col = _im2col(xn, batch, h, w, c, 2, "same")
    o = Guarded(col.shape[0], c)
    ops.gemm(col, pack_conv3x3(wt, DEV), bias=b, out=o.out)
    desc = f"downsample im2col+gemm B={batch} {h}x{w} c={c}"
    o.check(desc)
    ref = F.conv2d(x.float(), wt.float(), b, padding=1, stride=2).permute(0, 2, 3, 1).reshape(-1, c)
    err, note = gated(o.out, ref, 2e-3)
    return err, 2e-3, desc + note


def case_conv_im2col(batch, h, w, cin, cout, seed=0):
    """general-size 3x3 conv: explicit im2col (stride 1) + GEMM, for latents that do not tile into TMA boxes"""
    x = _rand(batch, cin, h, w, seed=seed).half()
    wt = _rand(cout, cin, 3, 3, seed=seed + 1, scale=(9 * cin) ** -0.5).half()
    b = _rand(cout, seed=seed + 2).float()
    from magicdance_b200.engine import pack_conv3x3
    xn = x.permute(0, 2, 3, 1).contiguous().reshape(batch * h * w, cin)
    col = _im2col(xn, batch, h, w, cin, 1, "same")
    o = Guarded(col.shape[0], cout)
    ops.gemm(col, pack_conv3x3(wt, DEV), bias=b, out=o.out)
    desc = f"conv3x3 im2col+gemm B={batch} {h}x{w} {cin}->{cout}"
    o.check(desc)
    ref = F.conv2d(x.float(), wt.float(), b, padding=1).permute(0, 2, 3, 1).reshape(-1, cout)
    err, note = gated(o.out, ref, 2e-3)
    return err, 2e-3, desc + note


def case_upsample(batch, h, w, c, seed=0):
    x = _rand(batch, c, h, w, seed=seed).half()
    xn = x.permute(0, 2, 3, 1).contiguous().reshape(batch * h * w, c)
    ptr = poisoned_alloc((batch * 4 * h * w, c), torch.float16)
    out = ops.upsample2x(xn, batch=batch, h=h, w=w, c=c)
    desc = f"upsample2x B={batch} {h}x{w} c={c}"
    check_poisoned(out, ptr, desc)
    ref = F.interpolate(x.float(), scale_factor=2, mode="nearest").permute(0, 2, 3, 1).reshape(-1, c)
    return rel(out.float(), ref), 0.0, desc


def case_groupnorm(batch, hw, c1, c2, eps, silu, mode=None, offset=0.3, seed=0):
    """mode: 0 auto, 1 two kernels (stats + last-CTA fold -> apply), 2 single-launch cluster kernel.
    offset: mean of the activations — a large value against a spread of ~1 is the catastrophic-cancellation case of
    E[x^2] - mean^2 that the pivot-shifted sums avoid.  Also checks run-to-run bit-equality (no atomics)."""
    x1 = (_rand(batch * hw, c1, seed=seed) * 1.5 + offset).half()
    x2 = (_rand(batch * hw, c2, seed=seed + 1) - 0.2 + offset).half() if c2 else None
    c = c1 + c2
    g = (1 + 0.1 * _rand(c, seed=seed + 2)).float()
    b = (0.1 * _rand(c, seed=seed + 3)).float()
    desc = f"groupnorm B={batch} hw={hw} c={c1}+{c2} silu={silu} mode={mode} offset={offset}"
    o1, o2 = Guarded(batch * hw, c, contiguous=True), Guarded(batch * hw, c, contiguous=True)
    out = ops.groupnorm(x1, g, b, batch=batch, hw=hw, eps=eps, silu=silu, x2=x2, mode=mode, out=o1.out)
    again = ops.groupnorm(x1, g, b, batch=batch, hw=hw, eps=eps, silu=silu, x2=x2, mode=mode, out=o2.out)
    o1.check(desc)
    o2.check(desc)
    xc = x1 if x2 is None else torch.cat([x1, x2], 1)
    xr = xc.double().reshape(batch, hw, c).permute(0, 2, 1)
    ref = F.group_norm(xr, 32, g.double(), b.double(), eps)
    if silu:
        ref = F.silu(ref)
    ref = ref.permute(0, 2, 1).reshape(batch * hw, c)
    err = rel(out.float(), ref)
    if not torch.equal(out, again):
        err = float("inf")  # non-deterministic
    return err, 2e-3, desc


def case_layernorm(rows, c, seed=0):
    x = (_rand(rows, c, seed=seed) * 2 + 0.5).half()
    g = (1 + 0.1 * _rand(c, seed=seed + 2)).float()
    b = (0.1 * _rand(c, seed=seed + 3)).float()
    o = Guarded(rows, c, contiguous=True)
    ops.layernorm(x, g, b, out=o.out)
    desc = f"layernorm rows={rows} c={c}"
    o.check(desc)
    ref = F.layer_norm(x.float(), (c,), g, b, 1e-5)
    return rel(o.out.float(), ref), 1.5e-3, desc


def _vt_cols(v, n, ldv, nb, pad):
    """V [nb*n, c] -> V^T [c, nb*ldv] in per-sample column blocks; the padding columns n..ldv of each hold `pad`"""
    vt = torch.full((v.shape[1], nb * ldv), pad, dtype=torch.float16, device=DEV)
    for b in range(nb):
        vt[:, b * ldv:b * ldv + n] = v[b * n:(b + 1) * n].t()
    return vt


def case_attention(batch, heads, d, nq, n0, n1=0, kv1_batches=1, bank_batches=None, ldv_pad=False, seed=0,
                   pad=0.0, kv0_shared=False, fused_qk=False, scale=None, sharp=False, lse=False):
    """Two-source attention into a guarded `out` (row pitch > heads*d).  pad: value of the V^T padding columns
    (n..ldv of every sample) and of the bank rows / columns of samples >= bank_batches, none of which may reach the
    output; q and k carry NaN row-stride padding.  kv0_shared: one source 0 for every sample (kv0_batches = 1, the
    text attention); fused_qk: q and k0 are the column halves of one [M, 2C] tensor (nq == n0); scale: explicit
    softmax scale; sharp: queries aligned with one key each — the last key of source 0 (its ragged tile) on even
    rows, a bank key on odd rows — for logits spread over ~10; lse: also the row log-sum-exp, against float64."""
    c = heads * d
    bb = batch if bank_batches is None else bank_batches
    kvb0 = 1 if kv0_shared else batch
    k0 = _rand(kvb0 * n0, c, seed=seed + 1).half()
    v0 = _rand(kvb0 * n0, c, seed=seed + 2).half()
    ldv = (n0 + 7) // 8 * 8 if ldv_pad else n0
    vt0 = _vt_cols(v0, n0, ldv, kvb0, pad)
    q = _rand(batch * nq, c, seed=seed).half()
    if n1:
        k1 = _rand(kv1_batches * n1, c, seed=seed + 3).half()
        v1 = _rand(kv1_batches * n1, c, seed=seed + 4).half()
        if kv1_batches > 1:  # the bank keys of samples without a bank must not be read
            k1[bb * n1:] = pad
        ldv1 = (n1 + 7) // 8 * 8
        vt1 = _vt_cols(v1, n1, ldv1, kv1_batches, pad)
        if kv1_batches > 1:
            vt1[:, bb * ldv1:] = pad
    if sharp:
        for b in range(batch):
            for i in range(nq):
                if i % 2 and n1 and b < bb:
                    tgt = k1[(b if kv1_batches > 1 else 0) * n1 + i % n1]
                else:
                    tgt = k0[(b if kvb0 > 1 else 0) * n0 + n0 - 1]
                q[b * nq + i] = (1.5 * tgt.float() + 0.5 * q[b * nq + i].float()).half()
    if fused_qk:
        assert nq == n0 and not kv0_shared
        qk = torch.cat([q, k0], 1)
        q, k0 = qk[:, :c], qk[:, c:]
    else:
        q, k0 = nan_padded(q), nan_padded(k0)
    kw = dict(ldv0_batch=ldv, kv0_batches=kvb0, scale=scale)
    if n1:
        kw.update(k1=nan_padded(k1), vt1=vt1, n1=n1, kv1_batches=kv1_batches, ldv1_batch=ldv1, bank_batches=bb)
    lg = Guarded(batch * heads, nq, torch.float32, contiguous=True) if lse else None
    desc = (f"attention B={batch} h={heads} d={d} nq={nq} n0={n0} n1={n1} kv1b={kv1_batches} bank_b={bb} pad={pad} "
            f"kv0_shared={kv0_shared} fused_qk={fused_qk} scale={scale} sharp={sharp}")
    out = guarded_run(batch * nq, c, lambda o: ops.attention(q, k0, vt0, n0, heads=heads, d=d, batch=batch, nq=nq,
                                                             out=o, lse=lg.out if lse else None, **kw), desc, True)
    dt = torch.float64 if lse else torch.float32
    sc = d ** -0.5 if scale is None else scale
    refs, lses = [], []
    for b in range(batch):
        qq = q[b * nq:(b + 1) * nq].to(dt).reshape(nq, heads, d).transpose(0, 1)
        k0b = b if kvb0 > 1 else 0
        kk = k0[k0b * n0:(k0b + 1) * n0].to(dt)
        vv = v0[k0b * n0:(k0b + 1) * n0].to(dt)
        if n1 and b < bb:
            sl = slice(b * n1, (b + 1) * n1) if kv1_batches > 1 else slice(0, n1)
            kk = torch.cat([kk, k1[sl].to(dt)], 0)
            vv = torch.cat([vv, v1[sl].to(dt)], 0)
        kk = kk.reshape(-1, heads, d).transpose(0, 1)
        vv = vv.reshape(-1, heads, d).transpose(0, 1)
        s = (qq @ kk.transpose(1, 2)) * sc
        refs.append((s.softmax(-1) @ vv).transpose(0, 1).reshape(nq, c))
        lses.append(s.logsumexp(-1))
    ref = torch.cat(refs, 0)
    err, note = gated(out, ref, 3e-3, rows=64, cols=d, groups=batch)
    if lse:
        lg.check(desc + " lse")
        e_lse = rel(lg.out, torch.cat(lses, 0))
        err, note = max(err, e_lse), note + f" lse rel-L2 {e_lse:.2e}"
    return err, 3e-3, desc + note


def case_time_path(batch, seed=0):
    base = [981, 441, 1, 999, 500, 21, 7, 123]
    t = torch.tensor([(base[i % 8] + 13 * (i // 8)) % 1000 for i in range(batch)], dtype=torch.long, device=DEV)
    ptr = poisoned_alloc((batch, 320), torch.float32)
    emb = ops.timestep_embedding(t, 320)
    check_poisoned(emb, ptr, "timestep embedding")
    half = 160
    freqs = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32, device=DEV) / half)
    args = t[:, None].float() * freqs[None]
    ref = torch.cat([torch.cos(args), torch.sin(args)], -1)
    e1 = float((emb - ref).abs().max())
    w = _rand(1280, 320, seed=seed, scale=320 ** -0.5).half()
    b = _rand(1280, seed=seed + 1).float()
    ptr = poisoned_alloc((batch, 1280), torch.float32)
    out = ops.skinny_linear(ref, w, b, silu_in=True, silu_out=True)
    check_poisoned(out, ptr, "skinny linear")
    r2 = F.silu(F.silu(ref) @ w.float().t() + b)
    return max(e1, rel(out, r2)), 1e-4, f"timestep embedding + skinny linear B={batch}"


def case_layout(batch, c, h, w, copies=1, seed=0):
    x = _rand(batch, c, h, w, seed=seed)
    desc = f"layout converts B={batch} c={c} {h}x{w} copies={copies}"
    o = Guarded(copies * batch * h * w, c, contiguous=True)
    y = ops.nchw_f32_to_nhwc_f16(x, out=o.out, copies=copies)
    o.check(desc + " nchw->nhwc")
    ref = x.half().permute(0, 2, 3, 1).reshape(-1, c).repeat(copies, 1)
    e1 = float((y.float() - ref.float()).abs().max())
    o2 = Guarded(batch * c * h, w, torch.float32, contiguous=True, shape=(batch, c, h, w))
    z = ops.nhwc_f16_to_nchw_f32(y[:batch * h * w], batch=batch, c=c, h=h, w=w, out=o2.out)
    o2.check(desc + " nhwc->nchw")
    e2 = float((z - x.half().float()).abs().max())
    return e1 + e2, 0.0, desc


def case_add(batch, n, bcast, alias=False, seed=0):
    """out = a + b; alias: out is a itself (the in-place residual add)"""
    a = _rand(batch, n, seed=seed).half()
    b = _rand(1 if bcast else batch, n, seed=seed + 1).half()
    ref = (a.float() + b.float()).half()
    desc = f"add B={batch} n={n} bcast={bcast} alias={alias}"
    o = Guarded(batch, n, contiguous=True)
    if alias:
        o.out.copy_(a)
        a = o.out
    ops.add(a, b, batch=batch, b_batches=1 if bcast else batch, out=o.out)
    o.check(desc)
    return float((o.out.float() - ref.float()).abs().max()), 0.0, desc


def case_cfg_ddim(shape=(2, 4, 64, 64), noise=False, sigma=0.0, update_x=False, seed=0):
    """classifier-free guidance + DDIM step (ddim.py p_sample_ddim) against float64; noise: the sigma * noise term
    (eta > 0); update_x: x advances in place and must equal x_prev bit for bit afterwards"""
    x, ec, eu = (_rand(*shape, seed=seed + i) for i in range(3))
    z = _rand(*shape, seed=seed + 3) if noise else None
    x0 = x.clone()
    a_t, a_prev, scale = 0.0047, 0.0058, 7.0
    coef = torch.tensor([scale, math.sqrt(a_t), math.sqrt(a_prev), math.sqrt(1 - a_prev - sigma ** 2), sigma,
                         math.sqrt(1 - a_t)], dtype=torch.float32, device=DEV)
    n = x.numel()
    o1 = Guarded(1, n, torch.float32, contiguous=True, bottom=8, shape=shape)
    o2 = Guarded(1, n, torch.float32, contiguous=True, bottom=8, shape=shape)
    xp, p0 = ops.cfg_ddim_update(x, ec, eu, coef, noise=z, x_prev=o1.out, pred_x0=o2.out, update_x=update_x)
    desc = f"cfg + ddim update {tuple(shape)} noise={noise} sigma={sigma} update_x={update_x}"
    o1.check(desc + " x_prev")
    o2.check(desc + " pred_x0")
    xd, ecd, eud = x0.double(), ec.double(), eu.double()
    e = eud + scale * (ecd - eud)
    rp0 = (xd - math.sqrt(1 - a_t) * e) / math.sqrt(a_t)
    rxp = math.sqrt(a_prev) * rp0 + math.sqrt(1 - a_prev - sigma ** 2) * e
    if noise:
        rxp = rxp + sigma * z.double()
    err = max(rel(xp, rxp), rel(p0, rp0))
    if not torch.equal(x, xp if update_x else x0):
        err = float("inf")
    return err, 1e-5, desc


NAN, INF = float("nan"), float("inf")

ALL_CASES = [
    (case_layout, (2, 4, 64, 64)),
    (case_layout, (1, 3, 256, 256)),
    (case_add, (2, 4096 * 320, False)),
    (case_add, (2, 64 * 1280, True)),
    (case_upsample, (2, 8, 8, 1280)),
    (case_time_path, (2,)),
    (case_time_path, (37,)),  # more rows than one skinny-linear launch holds (16)
    (case_cfg_ddim, ()),
    (case_layernorm, (4096, 320)),
    (case_layernorm, (300, 640)),
    (case_layernorm, (64, 1280)),
    (case_groupnorm, (2, 4096, 320, 0, 1e-5, True)),                 # auto: cluster of 4, 5 words per pixel
    (case_groupnorm, (1, 1024, 640, 320, 1e-5, True)),               # concat: groups straddle the two sources
    (case_groupnorm, (2, 64, 1280, 1280, 1e-5, True)),               # 8x8 level: one CTA per group
    (case_groupnorm, (2, 256, 1280, 0, 1e-6, False)),
    (case_groupnorm, (1, 16, 1280, 640, 1e-5, True)),
    (case_groupnorm, (2, 4096, 640, 320, 1e-5, True)),               # 960 channels at 64x64: the largest slice
    (case_groupnorm, (4, 1000, 320, 0, 1e-5, True)),                 # pixel count not a multiple of anything
    (case_groupnorm, (2, 4096, 320, 0, 1e-5, True, None, 40.0)),     # mean 40, spread 1.5: pivot-shifted variance
    (case_groupnorm, (16, 4096, 320, 0, 1e-5, True)),                # eight frames (cond+uncond), 10-channel groups: two kernels
    (case_groupnorm, (16, 1024, 1280, 640, 1e-5, True)),             # wide groups: the cluster kernel at every batch size
    (case_groupnorm, (25, 256, 1280, 0, 1e-6, False)),               # bank build: 25 timesteps
    (case_groupnorm, (16, 64, 1280, 1280, 1e-5, True)),
    (case_groupnorm, (16, 1024, 1280, 640, 1e-5, True, 1)),          # the same on the two-kernel path
    (case_groupnorm, (25, 256, 1280, 0, 1e-6, False, 1)),
    (case_groupnorm, (2, 4096, 320, 0, 1e-5, True, 1)),              # two-kernel path forced on small batches
    (case_groupnorm, (1, 1024, 640, 320, 1e-5, True, 1)),
    (case_groupnorm, (1, 16, 1280, 640, 1e-5, True, 1)),
    (case_groupnorm, (3, 1000, 320, 0, 1e-5, True, 1)),
    (case_groupnorm, (2, 4096, 128, 0, 1e-6, True, 1)),              # VAE: 4 channels per group
    (case_groupnorm, (8, 4096, 320, 0, 1e-5, True, 1, 40.0)),        # large mean on the two-kernel path
    (case_groupnorm, (16, 1024, 640, 0, 1e-5, True, 2)),             # cluster path forced on a large batch
    (case_groupnorm, (2, 16384, 128, 0, 1e-6, True, 2)),             # VAE widths on the cluster path
    (case_gemm, (128, 128, 64)),
    (case_gemm, (128, 160, 128)),
    (case_gemm, (4096, 320, 320, True, True)),
    (case_gemm, (1000, 640, 1280, True, False)),
    (case_gemm, (64, 1280, 2560, True, True)),
    (case_gemm, (77, 1280, 768)),
    (case_gemm, (320, 4096, 320)),
    (case_gemm, (64, 1280, 2560, True, True, 8)),
    (case_gemm, (256, 1280, 11520, True, False, 12)),
    (case_gemm, (256, 1280, 1280, True, True, 4)),
    (case_gemm, (1024, 640, 640, True, True, 2)),
    (case_gemm, (2048, 320, 1280, True, True, 2)),
    (case_gemm, (100, 1280, 2560, True, True, 8)),
    (case_gemm, (512, 1280, 5120, True, True, 0)),     # automatic: 160-wide tiles, 4 splits in a cluster
    (case_gemm, (512, 1280, 1280, True, True, 0)),     # automatic: 80-wide tiles, no split (short K)
    (case_gemm, (128, 1280, 2560, True, True, 0)),
    (case_gemm_ln, (8192, 320, 320)),                  # norm2 -> attn2.to_q at 64x64 (cond | uncond of one frame)
    (case_gemm_ln, (2048, 640, 640)),
    (case_gemm_ln, (512, 1280, 1280)),                 # 80-wide tiles: 16 CTAs recompute the same row statistics
    (case_gemm_ln, (100, 1280, 1280)),                 # ragged M
    (case_gemm_ln, (1024, 640, 640, 20.0)),            # row mean 20 against a spread of 1.3
    (case_gemm_batch_bias, (2, 1024, 640, 320)),
    (case_gemm_dual, (1024, 640, 640, 320)),
    (case_gemm_strided_out, (320, 77, 768)),
    (case_geglu, (4096, 320)),
    (case_geglu, (64, 1280)),
    (case_conv, (1, 64, 64, 320, 320)),
    (case_conv, (2, 32, 32, 640, 640, True, True)),
    (case_conv, (2, 16, 16, 1280, 1280)),
    (case_conv, (3, 8, 8, 1280, 1280, True, True)),
    (case_conv, (2, 4, 4, 1280, 1280)),
    (case_conv, (1, 8, 8, 2560, 1280, True, False, 8)),
    (case_conv, (2, 16, 16, 1280, 1280, True, True, 4)),
    (case_conv, (2, 32, 32, 640, 640, True, True, 2)),
    (case_conv, (1, 8, 256, 128, 128, True, True)),        # rows wider than the 128-pixel tile (VAE levels): x0 != 0
    (case_conv, (1, 4, 512, 128, 64, True, False)),
    (case_tuned, (PAIR, case_conv, 2, 6, 256, 64, 128, True, True)),
    (case_conv, (2, 16, 16, 1280, 1280, True, True, 0)),   # automatic: long K -> 160-wide tiles, 4 splits
    (case_conv, (2, 8, 8, 2560, 1280, True, True, 0)),     # automatic: 8 splits
    (case_conv, (1, 16, 16, 1280, 1280, True, False, 0)),  # ControlNet at one frame: M = 256
    # ---- the large-grid GEMM tiles forced onto small and odd problems ----
    (case_tuned, (PAIR, case_gemm, 512, 256, 128)),                       # K of 2 chunks: too little work even when forced
    (case_tuned, (PAIR, case_gemm, 384, 320, 320, True, True)),           # odd M tiles, 160-wide deep ring; bias+residual
    (case_tuned, (PAIR, case_gemm, 1000, 640, 1280, True, False)),        # ragged M: rows >= M of the last tile not stored
    (case_tuned, (PAIR, case_gemm, 300, 384, 192, True, True)),           # 128-wide deep-ring tiles
    (case_tuned, (PAIR, case_gemm, 4096, 320, 2880, True, True)),         # long K: the 6-stage ring wraps many times
    (case_tuned, (PAIR, case_gemm, 65536, 320, 320, True, True)),         # 512 M tiles x 2 N tiles, 160-wide
    (case_tuned, (PAIR, case_gemm, 4096, 1280, 640, True, True)),         # 256-wide tiles, 5 N tiles
    (case_tuned, (PAIR, case_gemm, 4096, 1280, 1280, True, True)),        # 256-wide tiles, K = 1280
    (case_tuned, (PAIR, case_gemm, 1000, 640, 2560, True, True)),         # 160-wide, ragged M, long K
    (case_tuned, (PAIR, case_gemm, 520, 200, 128, True, True)),           # N = 200: 128-wide tiles, the last chunk 8 columns wide
    (case_tuned, (PAIR, case_gemm_batch_bias, 2, 1024, 640, 320)),
    (case_tuned, (PAIR, case_gemm_dual, 1024, 640, 640, 320)),
    (case_tuned, (PAIR, case_gemm_strided_out, 320, 80, 768)),            # output row pitch > N
    (case_tuned, (PAIR, case_geglu, 512, 320)),
    (case_tuned, (PAIR, case_geglu, 4096, 320)),
    (case_tuned, (PAIR, case_conv, 1, 64, 64, 320, 320)),
    (case_tuned, (PAIR, case_conv, 8, 64, 64, 320, 320, True, True)),     # eight frames at 64x64: 256 M tiles, 160-wide
    (case_tuned, (PAIR, case_conv, 2, 32, 32, 640, 640, True, True)),
    (case_tuned, (PAIR, case_conv, 3, 8, 8, 1280, 1280, True, True)),     # 192 rows: the second M tile half out of range
    (case_tuned, (PAIR, case_conv, 16, 16, 16, 1280, 1280)),
    # ---- the same large shapes on the small-grid tiles (what the heuristics would not pick) ----
    (case_tuned, (NOPAIR, case_gemm, 65536, 320, 320, True, True)),
    (case_tuned, (NOPAIR, case_conv, 8, 64, 64, 320, 320, True, True)),
    (case_conv_direct, (1, 64, 64, 4, 320, 1, False, True)),
    (case_conv_direct, (2, 64, 64, 320, 4, 1, False)),
    (case_conv_direct, (1, 256, 256, 3, 16, 1, True)),
    (case_conv_direct, (1, 128, 128, 16, 32, 2, True)),
    (case_conv_direct, (1, 64, 64, 96, 256, 2, True)),
    (case_conv_s2, (2, 64, 64, 320, 320)),        # the three Downsample convs of one frame (cond | uncond)
    (case_conv_s2, (2, 32, 32, 640, 640)),
    (case_conv_s2, (2, 16, 16, 1280, 1280)),       # 8x8 output: two images per 128-row tile
    (case_conv_s2, (1, 16, 16, 1280, 1280)),       # ControlNet at one frame: half a tile
    (case_tuned, (PAIR, case_conv_s2, 16, 64, 64, 320, 320)),   # eight frames: the large-grid tiles
    (case_down, (2, 32, 32, 640)),
    (case_down, (1, 24, 16, 640)),
    (case_conv_im2col, (1, 12, 8, 1280, 1280)),
    (case_conv_im2col, (2, 6, 10, 640, 320)),
    (case_attention, (1, 8, 40, 4096, 4096)),
    (case_attention, (2, 8, 40, 1024, 1024, 1024, 2)),
    (case_attention, (2, 8, 40, 1024, 1024, 1024, 1, 1)),
    (case_attention, (2, 8, 40, 1024, 77, 0, 1, None, True)),
    (case_attention, (2, 8, 80, 256, 256, 256, 1)),
    (case_attention, (1, 8, 40, 384, 384, 128, 1)),
    (case_attention, (2, 8, 80, 200, 200, 0, 1)),
    (case_attention, (1, 8, 160, 320, 320, 64, 1)),
    (case_attention, (2, 8, 80, 1024, 77, 0, 1, None, True)),
    (case_attention, (2, 8, 160, 64, 64, 64, 2)),
    (case_attention, (1, 8, 160, 16, 16, 16, 1)),
    (case_attention, (2, 8, 160, 256, 77, 0, 1, None, True)),
    # ---- d=40 on the register-capped variant at two CTAs per SM (what large grids get) ----
    (case_tuned, (ATT2Q, case_attention, 1, 8, 40, 4096, 4096)),
    (case_tuned, (ATT2Q, case_attention, 2, 8, 40, 1024, 1024, 1024, 2)),
    (case_tuned, (ATT2Q, case_attention, 2, 8, 40, 1024, 1024, 1024, 1, 1)),
    (case_tuned, (ATT2Q, case_attention, 2, 8, 40, 1024, 77, 0, 1, None, True)),
    (case_tuned, (ATT2Q, case_attention, 1, 8, 40, 384, 384, 128, 1)),
    (case_attention, (16, 8, 40, 2048, 2048, 2048, 1, 8)),   # 2048 CTAs: the heuristics pick the two-CTA-per-SM variant (>= 512)
    # ---- d=80 with the d=40 key set: d=80 has one variant (one CTA per SM), so these are ragged / odd Q-tile shapes
    # that also check the key leaves d=80 alone ----
    (case_tuned, (ATT2Q, case_attention, 2, 8, 80, 256, 256, 256, 1)),
    (case_tuned, (ATT2Q, case_attention, 2, 8, 80, 200, 200, 0, 1)),          # ragged: the second Q tile is partly empty
    (case_tuned, (ATT2Q, case_attention, 2, 8, 80, 1024, 77, 0, 1, None, True)),
    (case_tuned, (ATT2Q, case_attention, 1, 8, 80, 384, 384, 128, 1)),        # odd number of Q tiles
    (case_attention, (16, 8, 80, 1024, 1024, 1024, 1, 8)),   # 1024 CTAs: the eight-frame d=80 grid
    # ---- edges: every output guarded (tests/kernel_guard.py) ----
    # ragged M on the 80-wide (N = 320), 128-wide (N = 384) and 160-wide (forced) small-grid tiles
    *[(case_gemm, (m, 320, 256, True, True)) for m in (1, 64, 127, 129)],
    *[(case_gemm, (m, 384, 256, True, True)) for m in (1, 64, 127, 129)],
    *[(case_tuned, (BN160, case_gemm, m, 320, 256, True, True)) for m in (1, 64, 127, 129)],
    (case_tuned, (PAIR, case_gemm, 129, 320, 256, True, True)),   # two M tiles, the second holding one row
    (case_tuned, (PAIR, case_gemm, 255, 320, 256, True, True)),
    *[(case_gemm, (300, n, 128, True, True)) for n in (8, 72, 77, 200)],  # N tails, 77: the scalar store tail
    (case_gemm, (200, 320, 64, True, True)),           # K of one chunk
    (case_gemm, (256, 320, 1024, True, True)),         # 8 CTAs, 16 chunks: the deep 80-wide ring
    (case_gemm, (256, 384, 1024, True, True)),         # ... and the deep 128-wide ring
    *[(case_gemm, (256, 320, 1536, True, True, s)) for s in (3, 5, 6, 12)],  # workspace split-K
    (case_gemm, (256, 320, 384, True, True, 4)),       # 6 chunks: 4 splits round to 3 (workspace)
    (case_gemm, (256, 320, 1280, True, True, 8)),      # 20 chunks: 8 splits round to 7
    (case_gemm, (256, 320, 320, True, True, 8)),       # 5 chunks: 5 splits of one chunk
    (case_gemm_batch_bias, (4, 64, 320, 320)),         # rows_per_batch < 128: two / eight samples per tile
    (case_gemm_batch_bias, (8, 16, 320, 320)),
    (case_gemm_batch_bias, (2, 64, 1280, 2560, 4)),    # ... with split-K in a cluster
    (case_gemm_batch_bias, (8, 16, 640, 2560, 3)),     # ... and through the workspace
    (case_tuned, (PAIR, case_gemm_batch_bias, 4, 64, 320, 320)),
    (case_tuned, (PAIR, case_gemm_batch_bias, 16, 16, 320, 320)),
    (case_conv, (3, 8, 8, 1280, 1280, True, True, 0, True)),   # the 8x8 ResBlock conv: timestep bias, automatic split
    (case_conv, (4, 4, 4, 1280, 1280, True, False, 0, True)),  # 4x4: eight images per tile
    (case_gemm_dual, (256, 320, 384, 576, 2)),         # the k1 boundary (chunk 6) inside split 0 of 2
    (case_gemm_dual, (256, 320, 384, 576, 3)),         # ... inside split 1 of 3 (workspace)
    (case_geglu, (77, 320)),
    (case_geglu, (100, 320)),
    (case_tuned, (PAIR, case_geglu, 300, 320)),
    (case_gemm_ln, (1, 320, 320)),
    (case_gemm_ln, (129, 640, 640)),
    # implicit-GEMM conv: each pixel_box mode, cin = 64 (one chunk per tap), cout 64 / 200
    (case_conv, (1, 2, 256, 64, 64)),                  # rows wider than the tile
    (case_conv, (1, 3, 128, 64, 64)),                  # rows exactly as wide as the tile
    (case_conv, (1, 16, 16, 64, 200)),                 # several rows per tile
    (case_conv, (12, 4, 4, 64, 64, True, True)),       # eight images per tile, the last tile half full
    (case_conv_s2, (1, 32, 32, 64, 64)),
    (case_conv_s2, (12, 8, 8, 64, 64)),
    (case_conv_s2, (2, 15, 15, 64, 200)),              # odd input: 8x8 outputs
    # direct conv: the generic kernel (cin not a multiple of 16, cout < 32, odd images), smallcin, smallcout
    (case_conv_direct, (2, 13, 7, 3, 8, 1, True, True)),
    (case_conv_direct, (1, 9, 9, 20, 40, 2, False, True)),
    (case_conv_direct, (2, 13, 7, 40, 3, 1, True)),
    (case_conv_direct, (1, 9, 9, 40, 8, 1, False, True)),
    (case_conv_direct, (2, 13, 7, 20, 40, 2, True, True)),
    (case_conv_direct, (1, 9, 9, 3, 3, 2, True)),
    (case_conv_direct, (1, 13, 7, 4, 8, 1, False, True)),
    (case_conv_direct, (2, 9, 9, 4, 64, 1, True, True)),
    (case_conv_direct, (1, 13, 7, 8, 4, 1, False)),
    (case_conv_direct, (2, 9, 9, 128, 4, 1, True)),
    (case_conv_direct, (1, 64, 64, 128, 3, 1, False)),    # the VAE's conv_out
    # data movement, bit-exact
    (case_upsample, (2, 5, 7, 8)),
    (case_upsample, (1, 3, 9, 64)),
    (case_add, (3, 4104, False, True)),
    (case_add, (3, 4104, True, True)),
    (case_layout, (2, 4, 9, 13, 2)),
    (case_layout, (1, 3, 7, 5, 3)),
    (case_cfg_ddim, ((1, 4, 9, 13), True, 0.3)),          # 468 elements
    (case_cfg_ddim, ((1, 4, 9, 13), False, 0.0, True)),
    (case_cfg_ddim, ((2, 4, 9, 13), True, 0.3, True)),
    # attention: guarded out (ldo > heads*d), NaN / Inf in every padding it must not read, run twice
    *[c for d in (40, 80, 160) for c in (
        (case_attention, (2, 8, d, 128, 77, 0, 1, None, True, 0, NAN, True)),             # shared text source
        (case_attention, (2, 8, d, 200, 200, 0, 1, None, False, 0, 0.0, False, True)),    # q | k halves of one tensor
        (case_attention, (2, 8, d, 1, 1, 1, 2, None, True, 0, NAN)),
        (case_attention, (2, 8, d, 63, 63, 65, 2, 1, True, 0, NAN)),                      # sample 1 has no bank
        (case_attention, (1, 8, d, 65, 65, 0, 1, None, True, 0, INF)),
        (case_attention, (2, 8, d, 129, 65, 65, 2, None, True, 0, NAN, False, False, 0.2)),
        (case_attention, (2, 1, d, 100, 77, 64, 2, None, True, 0, NAN)),                  # one head
        (case_attention, (2, 8, d, 129, 77, 64, 2, None, True, 0, NAN, False, False, None, True, True)),
        (case_attention, (1, 8, d, 63, 63, 65, 1, None, True, 0, NAN, False, False, None, False, True)),
    )],
    (case_tuned, (ATT2Q, case_attention, 2, 8, 40, 128, 77, 0, 1, None, True, 0, NAN, True)),
    (case_tuned, (ATT2Q, case_attention, 2, 8, 40, 63, 63, 65, 2, 1, True, 0, NAN)),
    (case_tuned, (ATT2Q, case_attention, 2, 8, 40, 129, 77, 64, 2, None, True, 0, NAN, False, False, None, True,
                  True)),
]
