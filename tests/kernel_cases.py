"""Per-kernel numerics cases: each function runs one C-ABI kernel on the GPU and returns
(error, tolerance, description) against a plain PyTorch fp32 reference of the same op computed
from the SAME fp16-rounded inputs.  Shared by tests/test_kernels_gpu.py and scripts/gpu_diag.py."""
import math

import torch
import torch.nn.functional as F

from magicdance_b200 import ops

DEV = "cuda"


def rel(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    return float((a - b).norm() / (b.norm() + 1e-30))


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def case_gemm(m, n, k, bias=False, residual=False, splits=1, seed=0):
    a = _rand(m, k, seed=seed).half()
    w = _rand(n, k, seed=seed + 1, scale=k ** -0.5).half()
    b = _rand(n, seed=seed + 2).float() if bias else None
    r = _rand(m, n, seed=seed + 3).half() if residual else None
    out = ops.gemm(a, w, bias=b, residual=r, splits=splits)
    ref = a.float() @ w.float().t()
    if bias:
        ref = ref + b
    if residual:
        ref = ref + r.float()
    return rel(out.float(), ref), 2e-3, f"gemm m={m} n={n} k={k} bias={bias} res={residual} splits={splits}"


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


def case_gemm_ln(m, n, k, offset=0.5, seed=0):
    """LayerNorm folded into the GEMM (ops.gemm(ln_u=...), engine.fold_layernorm) against LayerNorm -> Linear in fp32;
    offset: row mean of the activations (the correction rstd (acc - mean u) must not cancel)."""
    from magicdance_b200.engine import fold_layernorm
    x = (_rand(m, k, seed=seed) * 1.3 + offset).half()
    w = _rand(n, k, seed=seed + 1, scale=k ** -0.5)
    gamma = 1 + 0.1 * _rand(k, seed=seed + 2)
    beta = 0.1 * _rand(k, seed=seed + 3)
    b = 0.1 * _rand(n, seed=seed + 4)
    w_ln, u, v = fold_layernorm(w, gamma, beta, b, DEV)
    out = ops.gemm(x, w_ln, bias=v, ln_u=u, ln_eps=1e-5)
    ref = F.layer_norm(x.double(), (k,), gamma.double(), beta.double(), 1e-5) @ w.double().t() + b.double()
    return rel(out.float(), ref), 3e-3, f"gemm with folded LayerNorm m={m} n={n} k={k} offset={offset}"


def case_gemm_batch_bias(batch, hw, n, k, seed=0):
    m = batch * hw
    a = _rand(m, k, seed=seed).half()
    w = _rand(n, k, seed=seed + 1, scale=k ** -0.5).half()
    ball = _rand(batch, n + 64, seed=seed + 2).float()
    bias = ball[:, 32:32 + n]
    out = ops.gemm(a, w, bias=bias, bias_batch_stride=ball.stride(0), rows_per_batch=hw)
    ref = (a.float() @ w.float().t()).reshape(batch, hw, n) + bias[:, None, :]
    return rel(out.float(), ref.reshape(m, n)), 2e-3, f"gemm per-batch bias B={batch} hw={hw} n={n} k={k}"


def case_gemm_dual(m, n, k1, k2, seed=0):
    a1 = _rand(m, k1, seed=seed).half()
    a2 = _rand(m, k2, seed=seed + 5).half()
    w = _rand(n, k1 + k2, seed=seed + 1, scale=(k1 + k2) ** -0.5).half()
    out = ops.gemm(a1, w, a2=a2)
    ref = torch.cat([a1, a2], 1).float() @ w.float().t()
    return rel(out.float(), ref), 2e-3, f"gemm dual-source m={m} n={n} k={k1}+{k2}"


def case_gemm_strided_out(m, n, k, seed=0):
    """D written into a column slice of a wider, zero-initialised buffer (text V^T layout)."""
    a = _rand(m, k, seed=seed).half()
    w = _rand(n, k, seed=seed + 1, scale=k ** -0.5).half()
    ld = (n + 7) // 8 * 8
    buf = torch.zeros(m, 2 * ld, dtype=torch.float16, device=DEV)
    ops.gemm(a, w, out=buf[:, ld:ld + n])
    ref = a.float() @ w.float().t()
    untouched = float(buf[:, :ld].abs().max()) + (float(buf[:, ld + n:].abs().max()) if ld > n else 0.0)
    return rel(buf[:, ld:ld + n].float(), ref) + untouched, 2e-3, f"gemm strided out m={m} n={n} k={k}"


def case_geglu(m, c, seed=0):
    from magicdance_b200.engine import pack_geglu
    x = _rand(m, c, seed=seed).half()
    w = _rand(8 * c, c, seed=seed + 1, scale=c ** -0.5)
    b = _rand(8 * c, seed=seed + 2, scale=0.1)
    wp, bp = pack_geglu(w, b, DEV)
    out = ops.gemm(x, wp, bias=bp, epilogue=ops.EPI_GEGLU)
    y = x.float() @ w.half().float().t() + b
    v, g = y.chunk(2, dim=-1)
    ref = v * F.gelu(g)
    return rel(out.float(), ref), 3e-3, f"geglu m={m} c={c}"


def case_conv(batch, h, w, cin, cout, bias=True, residual=False, splits=1, seed=0):
    x = _rand(batch, cin, h, w, seed=seed).half()
    wt = _rand(cout, cin, 3, 3, seed=seed + 1, scale=(9 * cin) ** -0.5).half()
    b = _rand(cout, seed=seed + 2).float() if bias else None
    from magicdance_b200.engine import pack_conv3x3
    xn = x.permute(0, 2, 3, 1).contiguous().reshape(batch * h * w, cin)
    r = _rand(batch * h * w, cout, seed=seed + 3).half() if residual else None
    out = ops.gemm(xn, pack_conv3x3(wt, DEV), bias=b, residual=r, conv=(batch, h, w, cin), splits=splits)
    ref = F.conv2d(x.float(), wt.float(), b, padding=1).permute(0, 2, 3, 1).reshape(batch * h * w, cout)
    if residual:
        ref = ref + r.float()
    return rel(out.float(), ref), 2e-3, f"conv3x3 igemm B={batch} {h}x{w} {cin}->{cout} splits={splits}"


def case_conv_s2(batch, h, w, cin, cout, seed=0):
    """3x3 stride-2 pad-1 conv (Downsample.op, openaimodel.py:175) as implicit GEMM: TMA element strides of 2"""
    x = _rand(batch * h * w, cin, seed=seed).half()
    wt = _rand(cout, 3, 3, cin, seed=seed + 1, scale=(9 * cin) ** -0.5).half()
    b = _rand(cout, seed=seed + 2).float()
    out = ops.gemm(x, wt.reshape(cout, 9 * cin), bias=b, conv=(batch, h, w, cin), conv_stride=2)
    xr = x.float().reshape(batch, h, w, cin).permute(0, 3, 1, 2)
    ref = F.conv2d(xr, wt.float().permute(0, 3, 1, 2), b, stride=2, padding=1).permute(0, 2, 3, 1).reshape(-1, cout)
    return rel(out.float(), ref), 2e-3, f"conv 3x3 stride 2 (implicit GEMM) B={batch} {h}x{w} {cin}->{cout}"


def case_conv_direct(batch, h, w, cin, cout, stride, silu, residual=False, seed=0):
    x = _rand(batch, cin, h, w, seed=seed).half()
    wt = _rand(cout, cin, 3, 3, seed=seed + 1, scale=(9 * cin) ** -0.5).half()
    b = _rand(cout, seed=seed + 2).float()
    from magicdance_b200.engine import pack_conv3x3
    xn = x.permute(0, 2, 3, 1).contiguous().reshape(batch * h * w, cin)
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    r = _rand(batch * ho * wo, cout, seed=seed + 3).half() if residual else None
    out = ops.conv3x3_direct(xn, pack_conv3x3(wt, DEV), b, batch=batch, h=h, w=w, cin=cin, cout=cout, stride=stride,
                             silu=silu, residual=r)
    ref = F.conv2d(x.float(), wt.float(), b, padding=1, stride=stride)
    if silu:
        ref = F.silu(ref)
    ref = ref.permute(0, 2, 3, 1).reshape(batch * ho * wo, cout)
    if residual:
        ref = ref + r.float()
    return rel(out.float(), ref), 2e-3, f"conv3x3 direct B={batch} {h}x{w} {cin}->{cout} s={stride} silu={silu}"


def case_down(batch, h, w, c, seed=0):
    x = _rand(batch, c, h, w, seed=seed).half()
    wt = _rand(c, c, 3, 3, seed=seed + 1, scale=(9 * c) ** -0.5).half()
    b = _rand(c, seed=seed + 2).float()
    from magicdance_b200.engine import pack_conv3x3
    xn = x.permute(0, 2, 3, 1).contiguous().reshape(batch * h * w, c)
    col = ops.im2col3x3(xn, batch=batch, h=h, w=w, c=c, stride=2)
    out = ops.gemm(col, pack_conv3x3(wt, DEV), bias=b)
    ref = F.conv2d(x.float(), wt.float(), b, padding=1, stride=2).permute(0, 2, 3, 1).reshape(-1, c)
    return rel(out.float(), ref), 2e-3, f"downsample im2col+gemm B={batch} {h}x{w} c={c}"


def case_conv_im2col(batch, h, w, cin, cout, seed=0):
    """general-size 3x3 conv: explicit im2col (stride 1) + GEMM, for latents that do not tile into TMA boxes"""
    x = _rand(batch, cin, h, w, seed=seed).half()
    wt = _rand(cout, cin, 3, 3, seed=seed + 1, scale=(9 * cin) ** -0.5).half()
    b = _rand(cout, seed=seed + 2).float()
    from magicdance_b200.engine import pack_conv3x3
    xn = x.permute(0, 2, 3, 1).contiguous().reshape(batch * h * w, cin)
    col = ops.im2col3x3(xn, batch=batch, h=h, w=w, c=cin, stride=1)
    out = ops.gemm(col, pack_conv3x3(wt, DEV), bias=b)
    ref = F.conv2d(x.float(), wt.float(), b, padding=1).permute(0, 2, 3, 1).reshape(-1, cout)
    return rel(out.float(), ref), 2e-3, f"conv3x3 im2col+gemm B={batch} {h}x{w} {cin}->{cout}"


def case_upsample(batch, h, w, c, seed=0):
    x = _rand(batch, c, h, w, seed=seed).half()
    xn = x.permute(0, 2, 3, 1).contiguous().reshape(batch * h * w, c)
    out = ops.upsample2x(xn, batch=batch, h=h, w=w, c=c)
    ref = F.interpolate(x.float(), scale_factor=2, mode="nearest").permute(0, 2, 3, 1).reshape(-1, c)
    return rel(out.float(), ref), 0.0, f"upsample2x B={batch} {h}x{w} c={c}"


def case_groupnorm(batch, hw, c1, c2, eps, silu, mode=None, offset=0.3, seed=0):
    """mode: 0 auto, 1 two kernels (stats + last-CTA fold -> apply), 2 single-launch cluster kernel.
    offset: mean of the activations — a large value against a spread of ~1 is the catastrophic-cancellation case of
    E[x^2] - mean^2 that the pivot-shifted sums avoid.  Also checks run-to-run bit-equality (no atomics)."""
    x1 = (_rand(batch * hw, c1, seed=seed) * 1.5 + offset).half()
    x2 = (_rand(batch * hw, c2, seed=seed + 1) - 0.2 + offset).half() if c2 else None
    c = c1 + c2
    g = (1 + 0.1 * _rand(c, seed=seed + 2)).float()
    b = (0.1 * _rand(c, seed=seed + 3)).float()
    out = ops.groupnorm(x1, g, b, batch=batch, hw=hw, eps=eps, silu=silu, x2=x2, mode=mode)
    again = ops.groupnorm(x1, g, b, batch=batch, hw=hw, eps=eps, silu=silu, x2=x2, mode=mode)
    xc = x1 if x2 is None else torch.cat([x1, x2], 1)
    xr = xc.double().reshape(batch, hw, c).permute(0, 2, 1)
    ref = F.group_norm(xr, 32, g.double(), b.double(), eps)
    if silu:
        ref = F.silu(ref)
    ref = ref.permute(0, 2, 1).reshape(batch * hw, c)
    err = rel(out.float(), ref)
    if not torch.equal(out, again):
        err = float("inf")  # non-deterministic
    return err, 2e-3, f"groupnorm B={batch} hw={hw} c={c1}+{c2} silu={silu} mode={mode} offset={offset}"


def case_layernorm(rows, c, seed=0):
    x = (_rand(rows, c, seed=seed) * 2 + 0.5).half()
    g = (1 + 0.1 * _rand(c, seed=seed + 2)).float()
    b = (0.1 * _rand(c, seed=seed + 3)).float()
    out = ops.layernorm(x, g, b)
    ref = F.layer_norm(x.float(), (c,), g, b, 1e-5)
    return rel(out.float(), ref), 1.5e-3, f"layernorm rows={rows} c={c}"


def case_attention(batch, heads, d, nq, n0, n1=0, kv1_batches=1, bank_batches=None, ldv_pad=False, seed=0):
    c = heads * d
    q = _rand(batch * nq, c, seed=seed).half()
    k0 = _rand(batch * n0, c, seed=seed + 1).half()
    v0 = _rand(batch * n0, c, seed=seed + 2).half()
    ldv = (n0 + 7) // 8 * 8 if ldv_pad else n0
    vt0 = torch.zeros(c, batch * ldv, dtype=torch.float16, device=DEV)
    for b in range(batch):
        vt0[:, b * ldv:b * ldv + n0] = v0[b * n0:(b + 1) * n0].t()
    kw = {}
    if n1:
        k1 = _rand(kv1_batches * n1, c, seed=seed + 3).half()
        v1 = _rand(kv1_batches * n1, c, seed=seed + 4).half()
        kw = dict(k1=k1, vt1=v1.t().contiguous(), n1=n1, kv1_batches=kv1_batches,
                  bank_batches=batch if bank_batches is None else bank_batches)
    out = ops.attention(q, k0, vt0, n0, heads=heads, d=d, batch=batch, nq=nq, ldv0_batch=ldv, **kw)
    refs = []
    bb = batch if bank_batches is None else bank_batches
    for b in range(batch):
        qq = q[b * nq:(b + 1) * nq].float().reshape(nq, heads, d).transpose(0, 1)
        kk = k0[b * n0:(b + 1) * n0].float()
        vv = v0[b * n0:(b + 1) * n0].float()
        if n1 and b < bb:
            sl = slice(b * n1, (b + 1) * n1) if kv1_batches > 1 else slice(0, n1)
            kk = torch.cat([kk, k1[sl].float()], 0)
            vv = torch.cat([vv, v1[sl].float()], 0)
        kk = kk.reshape(-1, heads, d).transpose(0, 1)
        vv = vv.reshape(-1, heads, d).transpose(0, 1)
        s = (qq @ kk.transpose(1, 2)) * d ** -0.5
        o = s.softmax(-1) @ vv
        refs.append(o.transpose(0, 1).reshape(nq, c))
    ref = torch.cat(refs, 0)
    return rel(out.float(), ref), 3e-3, (f"attention B={batch} h={heads} d={d} nq={nq} n0={n0} n1={n1} "
                                          f"kv1b={kv1_batches} bank_b={bb}")


def case_time_path(batch, seed=0):
    base = [981, 441, 1, 999, 500, 21, 7, 123]
    t = torch.tensor([(base[i % 8] + 13 * (i // 8)) % 1000 for i in range(batch)], dtype=torch.long, device=DEV)
    emb = ops.timestep_embedding(t, 320)
    half = 160
    freqs = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32, device=DEV) / half)
    args = t[:, None].float() * freqs[None]
    ref = torch.cat([torch.cos(args), torch.sin(args)], -1)
    e1 = float((emb - ref).abs().max())
    w = _rand(1280, 320, seed=seed, scale=320 ** -0.5).half()
    b = _rand(1280, seed=seed + 1).float()
    out = ops.skinny_linear(ref, w, b, silu_in=True, silu_out=True)
    r2 = F.silu(F.silu(ref) @ w.float().t() + b)
    return max(e1, rel(out, r2)), 1e-4, f"timestep embedding + skinny linear B={batch}"


def case_layout(batch, c, h, w, seed=0):
    x = _rand(batch, c, h, w, seed=seed)
    y = ops.nchw_f32_to_nhwc_f16(x)
    ref = x.half().permute(0, 2, 3, 1).reshape(-1, c)
    e1 = float((y.float() - ref.float()).abs().max())
    z = ops.nhwc_f16_to_nchw_f32(y, batch=batch, c=c, h=h, w=w)
    e2 = float((z - x.half().float()).abs().max())
    return e1 + e2, 0.0, f"layout converts B={batch} c={c} {h}x{w}"


def case_add(batch, n, bcast, seed=0):
    a = _rand(batch, n, seed=seed).half()
    b = _rand(1 if bcast else batch, n, seed=seed + 1).half()
    out = ops.add(a, b, batch=batch, b_batches=1 if bcast else batch)
    ref = (a.float() + b.float()).half()
    return float((out.float() - ref.float()).abs().max()), 0.0, f"add B={batch} n={n} bcast={bcast}"


def case_cfg_ddim(seed=0):
    x, ec, eu = (_rand(2, 4, 64, 64, seed=seed + i) for i in range(3))
    a_t, a_prev, sigma, scale = 0.0047, 0.0058, 0.0, 7.0
    coef = torch.tensor([scale, math.sqrt(a_t), math.sqrt(a_prev), math.sqrt(1 - a_prev - sigma ** 2), sigma,
                         math.sqrt(1 - a_t)], dtype=torch.float32, device=DEV)
    xp, p0 = ops.cfg_ddim_update(x, ec, eu, coef)
    e = eu + scale * (ec - eu)
    rp0 = (x - math.sqrt(1 - a_t) * e) / math.sqrt(a_t)
    rxp = math.sqrt(a_prev) * rp0 + math.sqrt(1 - a_prev) * e
    return max(rel(xp, rxp), rel(p0, rp0)), 1e-5, "cfg + ddim update"


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
]
