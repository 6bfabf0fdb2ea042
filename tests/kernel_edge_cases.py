"""Edge cases of the small kernels that tests/kernel_cases.py has no case function for: softmax_rows (VAE attention),
im2col3x3 in both paddings, timestep_embedding, skinny_linear, and the implicit-GEMM conv's refusal of wide rows at
stride 2.  Same (error, tolerance, description) contract and the same output poisoning (tests/kernel_guard.py);
references in float64 or, for data movement, bit-exact.  Run by tests/test_kernel_edges_gpu.py."""
import math

import torch
import torch.nn.functional as F

from magicdance_b200 import ops
from tests.kernel_cases import DEV, _rand, rel
from tests.kernel_guard import Guarded, check_poisoned, poisoned_alloc


def case_softmax_rows(rows, cols, ld_extra, scale, amp=1.0, seed=0):
    """in-place row softmax of a [rows, cols] view whose row stride exceeds cols by ld_extra + 8: the columns between
    cols and the stride (guards) must stay untouched.  amp scales the inputs (x 8 with scale 4: a sharp softmax)."""
    x = (_rand(rows, cols, seed=seed) * amp).half()
    o = Guarded(rows, cols, right=ld_extra)
    o.out.copy_(x)
    ops.softmax_rows(o.out, scale)
    desc = f"softmax_rows {rows}x{cols} ld={o.out.stride(0)} scale={scale} amp={amp}"
    o.check(desc)
    return rel(o.out, torch.softmax(x.double() * scale, 1)), 2e-3, desc


def case_im2col(batch, h, w, c, stride, pad):
    """ops.im2col3x3 bit-exact against slicing the padded NHWC input (pad 'same': one halo pixel on every side; 'br':
    one at the bottom / right), columns tap-major (kh, kw, channel)"""
    x = _rand(batch, h, w, c).half()
    xp = F.pad(x, (0, 0, 1, 1, 1, 1) if pad == "same" else (0, 0, 0, 1, 0, 1))
    ho, wo = (xp.shape[1] - 3) // stride + 1, (xp.shape[2] - 3) // stride + 1
    taps = [xp[:, kh:kh + stride * (ho - 1) + 1:stride, kw:kw + stride * (wo - 1) + 1:stride] for kh in range(3)
            for kw in range(3)]
    ref = torch.stack(taps, 3).reshape(batch * ho * wo, 9 * c)
    ptr = poisoned_alloc(ref.shape, torch.float16)
    col = ops.im2col3x3(x.reshape(-1, c), batch=batch, h=h, w=w, c=c, stride=stride, pad=pad)
    desc = f"im2col3x3 B={batch} {h}x{w} c={c} stride={stride} pad={pad}"
    check_poisoned(col, ptr, desc)
    return 0.0 if torch.equal(col, ref) else float("inf"), 0.0, desc


def case_timestep_embedding(ts, rows):
    """sinusoidal embedding (320 channels) of t against float64; rows > len(t): row b uses t[b % len(t)].  The fp32
    argument t * freq of up to 999 rad carries a rounding error of a few 1e-5, hence the tolerance."""
    t = torch.tensor(ts, dtype=torch.long, device=DEV)
    ptr = poisoned_alloc((rows, 320), torch.float32)
    emb = ops.timestep_embedding(t, 320, rows)
    desc = f"timestep_embedding t={ts} rows={rows}"
    check_poisoned(emb, ptr, desc)
    freqs = torch.exp(-math.log(10000) * torch.arange(160, dtype=torch.float64, device=DEV) / 160)
    args = t.double()[torch.arange(rows, device=DEV) % len(ts), None] * freqs[None]
    ref = torch.cat([torch.cos(args), torch.sin(args)], -1)
    return float((emb.double() - ref).abs().max()), 3e-4, desc


def case_skinny_linear(rows, k, n, bias, silu_in, silu_out, seed=0):
    """out = silu?(silu?(x) W^T + b) for a handful of rows (the timestep MLP) against float64; rows > 16 go through
    ops' 16-row chunks, and 1-2 / 3-8 / 9-16 rows through different kernel instantiations"""
    x = _rand(rows, k, seed=seed)
    w = _rand(n, k, seed=seed + 1, scale=k ** -0.5).half()
    b = _rand(n, seed=seed + 2) if bias else None
    ptr = poisoned_alloc((rows, n), torch.float32)
    out = ops.skinny_linear(x, w, b, silu_in=silu_in, silu_out=silu_out)
    desc = f"skinny_linear rows={rows} k={k} n={n} bias={bias} silu_in={silu_in} silu_out={silu_out}"
    check_poisoned(out, ptr, desc)
    xd = F.silu(x.double()) if silu_in else x.double()
    ref = xd @ w.double().t() + (b.double() if bias else 0.0)
    if silu_out:
        ref = F.silu(ref)
    return rel(out, ref), 1e-4, desc


def case_conv_s2_wide_rows_rejected():
    """stride-2 implicit GEMM whose output rows are wider than the 128-pixel tile: refused with a message, nothing
    launched"""
    x = torch.zeros(2 * 512, 64, dtype=torch.float16, device=DEV)
    w = torch.zeros(64, 9 * 64, dtype=torch.float16, device=DEV)
    n0 = ops.launch_count()
    try:
        ops.gemm(x, w, conv=(1, 2, 512, 64), conv_stride=2)
    except RuntimeError as e:
        ok = "conv rows wider than 128 pixels need 128 | w and stride 1" in str(e) and ops.launch_count() == n0
        return 0.0 if ok else float("inf"), 0.0, f"stride-2 conv with 256-pixel output rows refused: {e}"
    return float("inf"), 0.0, "stride-2 conv with 256-pixel output rows was not refused"


_SILU = [(False, False), (True, False), (False, True), (True, True)]

EDGE_CASES = [
    *[(case_softmax_rows, (37, cols, 8, 0.05)) for cols in (8, 72, 4096, 4104)],
    *[(case_softmax_rows, (37, cols, 24, 4.0, 8.0)) for cols in (8, 72, 4096, 4104)],
    (case_im2col, (2, 7, 5, 8, 1, "same")),
    (case_im2col, (1, 9, 7, 16, 2, "same")),
    (case_im2col, (2, 7, 5, 8, 1, "br")),
    (case_im2col, (1, 9, 7, 16, 2, "br")),
    (case_im2col, (1, 2, 2, 8, 1, "br")),   # the smallest image the bottom / right padding takes
    (case_im2col, (3, 2, 2, 8, 2, "br")),
    (case_timestep_embedding, ((0, 999), 4)),
    (case_timestep_embedding, ((999, 0, 500), 6)),
    *[(case_skinny_linear, (rows, k, n, i % 2 == 0, *_SILU[(i + j) % 4]))
      for i, rows in enumerate((1, 2, 3, 8, 9, 16, 17)) for j, (k, n) in enumerate(((8, 77), (264, 1), (1280, 77)))],
    (case_conv_s2_wide_rows_rejected, ()),
]
