"""Launches the step's dominant kernels a few times each at their real shapes (B=1 frame, paired
cond/uncond batch of 2) so that `ncu --set full` can capture them without replaying a whole step."""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch  # noqa: E402
from magicdance_b200 import ops  # noqa: E402

D = "cuda"
h = lambda *s: torch.randn(*s, device=D).half()
f = lambda *s: torch.randn(*s, device=D)
ops.ensure_device()
flush = torch.empty(256 * 2 ** 20, dtype=torch.uint8, device=D)
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 2
for _ in range(reps):
    # self-attention of the paired batch at 64x64: sample 0 reads the bank (8192 keys), sample 1 does not
    q, k0, vt0 = h(2 * 4096, 320), h(2 * 4096, 320), h(320, 2 * 4096)
    k1, vt1 = h(4096, 320), h(320, 4096)
    flush.zero_()
    ops.attention(q, k0, vt0, 4096, heads=8, d=40, batch=2, nq=4096, k1=k1, vt1=vt1, n1=4096, kv1_batches=1, bank_batches=1)
    # 3x3 convs (implicit GEMM) of the paired batch
    for (b, hh, cin, cout) in ((2, 64, 320, 320), (2, 32, 640, 640), (2, 16, 1280, 1280), (2, 8, 1280, 1280)):
        x, w, bias = h(b * hh * hh, cin), h(cout, 9 * cin), f(cout)
        flush.zero_()
        ops.gemm(x, w, bias=bias, conv=(b, hh, hh, cin))
    # transformer linears
    for (m, n, k) in ((8192, 320, 320), (2048, 640, 640), (512, 1280, 1280), (8192, 320, 1280)):
        a, w, bias, r = h(m, k), h(n, k), f(n), h(m, n)
        flush.zero_()
        ops.gemm(a, w, bias=bias, residual=r)
    # group norms
    for (b, hw, c1, c2) in ((2, 4096, 320, 0), (2, 1024, 640, 640), (2, 64, 1280, 1280)):
        x1 = h(b * hw, c1)
        x2 = h(b * hw, c2) if c2 else None
        g_, b_ = f(c1 + c2), f(c1 + c2)
        flush.zero_()
        ops.groupnorm(x1, g_, b_, batch=b, hw=hw, eps=1e-5, silu=True, x2=x2)
    x, g_, b_ = h(8192, 320), f(320), f(320)
    ops.layernorm(x, g_, b_)
    # ---- eight frames per GPU (cond | uncond batch of 16): the large-grid GEMM tiles, the two-CTA-per-SM d=40 attention,
    # the two-kernel GroupNorm ----
    for (b, hh, cin, cout) in ((16, 32, 1280, 640), (16, 16, 1280, 1280), (16, 64, 320, 320)):
        x, w, bias = h(b * hh * hh, cin), h(cout, 9 * cin), f(cout)
        flush.zero_()
        ops.gemm(x, w, bias=bias, conv=(b, hh, hh, cin))
    for (m, n, k) in ((65536, 320, 320), (16384, 640, 640), (65536, 320, 1280)):
        a, w, bias, r = h(m, k), h(n, k), f(n), h(m, n)
        flush.zero_()
        ops.gemm(a, w, bias=bias, residual=r)
    from magicdance_b200.engine import pack_geglu
    x, (wp, bp) = h(65536, 320), pack_geglu(torch.randn(2560, 320), torch.randn(2560), D)
    flush.zero_()
    ops.gemm(x, wp, bias=bp, epilogue=ops.EPI_GEGLU)
    q, k0, vt0 = h(8 * 4096, 320), h(8 * 4096, 320), h(320, 8 * 4096)
    flush.zero_()
    ops.attention(q, k0, vt0, 4096, heads=8, d=40, batch=8, nq=4096, k1=k1, vt1=vt1, n1=4096, kv1_batches=1, bank_batches=8)
    x1, g_, b_ = h(16 * 4096, 320), f(320), f(320)
    flush.zero_()
    ops.groupnorm(x1, g_, b_, batch=16, hw=4096, eps=1e-5, silu=True)
torch.cuda.synchronize()
print("done")
