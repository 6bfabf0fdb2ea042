"""Per-kernel GPU time without profiler overhead: each case is captured `reps` times back to back
in a CUDA graph and the replay is timed with CUDA events (warm L2; launch latency hidden)."""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch  # noqa: E402
from magicdance_b200 import ops  # noqa: E402
from magicdance_b200.engine import pack_geglu  # noqa: E402

D = "cuda"
h = lambda *s: torch.randn(*s, device=D).half()
f = lambda *s: torch.randn(*s, device=D)


def timeit(name, fn, reps=20, flops=None, bytes_=None):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    best = 1e9
    for _ in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) * 1e3 / reps)
    extra = ""
    if flops:
        extra += f"  {flops / best / 1e6:8.1f} TFLOP/s"
    if bytes_:
        extra += f"  {bytes_ / best / 1e3:8.1f} GB/s"
    print(f"{name:58s} {best:9.2f} us{extra}", flush=True)


def gemm_case(m, n, k, splits=1, bias=True, res=True):
    a, w = h(m, k), h(n, k)
    b = f(n) if bias else None
    r = h(m, n) if res else None
    timeit(f"gemm m={m} n={n} k={k} splits={splits}", lambda: ops.gemm(a, w, bias=b, residual=r, splits=splits),
           flops=2.0 * m * n * k)


def conv_case(b, hh, ww, cin, cout, splits=1):
    x, w = h(b * hh * ww, cin), h(cout, 9 * cin)
    bias = f(cout)
    timeit(f"conv B={b} {hh}x{ww} {cin}->{cout} splits={splits}",
           lambda: ops.gemm(x, w, bias=bias, conv=(b, hh, ww, cin), splits=splits), flops=2.0 * b * hh * ww * cout * 9 * cin)


def attn_case(b, d, nq, n0, n1=0):
    c = 8 * d
    q, k0, vt0 = h(b * nq, c), h(b * n0, c), h(c, b * ((n0 + 7) // 8 * 8))
    kw = {}
    if n1:
        kw = dict(k1=h(n1, c), vt1=h(c, n1), n1=n1, kv1_batches=1, bank_batches=b)
    timeit(f"attention B={b} d={d} nq={nq} n0={n0} n1={n1}",
           lambda: ops.attention(q, k0, vt0, n0, heads=8, d=d, batch=b, nq=nq, ldv0_batch=(n0 + 7) // 8 * 8, **kw),
           flops=4.0 * b * 8 * nq * (n0 + n1) * d)


def timeit_eager(name, fn, reps=20, flops=None, bytes_=None):
    """CUDA events around `reps` eager calls (for torch autograd, which a CUDA graph cannot capture here)"""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    best = 1e9
    for _ in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) * 1e3 / reps)
    extra = f"  {flops / best / 1e6:8.1f} TFLOP/s" if flops else ""
    if bytes_:
        extra += f"  {bytes_ / best / 1e3:8.1f} GB/s"
    print(f"{name:58s} {best:9.2f} us{extra}", flush=True)


def attn_bwd_case(b, d, nq, n0, n1=0, heads=8):
    """forward-with-LSE and backward (ours) against torch SDPA forward + backward on the torch.cat'ed K / V.
    Algorithmic FLOP: forward 4 nq nk d, backward 10 nq nk d per head (nk = n0 + n1)."""
    import torch.nn.functional as F
    c = heads * d
    nk = n0 + n1
    ldv = (n0 + 7) // 8 * 8
    q, k0, vt0, dout = h(b * nq, c), h(b * n0, c), h(c, b * ldv), h(b * nq, c)
    kw = dict(heads=heads, d=d, batch=b, nq=nq, ldv0_batch=ldv)
    if n1:
        kw.update(k1=h(b * n1, c), vt1=h(c, b * n1), n1=n1, kv1_batches=b, bank_batches=b)
    lse = torch.empty(b, heads, nq, device=D)
    out = ops.attention(q, k0, vt0, n0, lse=lse, **kw)
    fl_f, fl_b = 4.0 * b * heads * nq * nk * d, 10.0 * b * heads * nq * nk * d
    tag = f"B={b} d={d} nq={nq} n0={n0} n1={n1}"
    timeit(f"ours fwd+lse {tag}", lambda: ops.attention(q, k0, vt0, n0, out=out, lse=lse, **kw), flops=fl_f)
    timeit(f"ours bwd     {tag}", lambda: ops.attention_backward(q, k0, vt0, n0, out, dout, lse, **kw), flops=fl_b)
    # torch: [B, heads, tokens, d] with the two sources concatenated
    qt = torch.randn(b, heads, nq, d, device=D, dtype=torch.float16, requires_grad=True)
    kt = torch.randn(b, heads, nk, d, device=D, dtype=torch.float16, requires_grad=True)
    vt = torch.randn(b, heads, nk, d, device=D, dtype=torch.float16, requires_grad=True)
    g = torch.randn(b, heads, nq, d, device=D, dtype=torch.float16)
    with torch.no_grad():
        timeit_eager(f"sdpa fwd     {tag}", lambda: F.scaled_dot_product_attention(qt, kt, vt), flops=fl_f)
    timeit_eager(f"sdpa fwd+bwd {tag}",
                 lambda: torch.autograd.grad(F.scaled_dot_product_attention(qt, kt, vt), (qt, kt, vt), g),
                 flops=fl_f + fl_b)


def gemm_bwd_case(m, n, k, conv=None, stride=1):
    """our dA, dW and dbias (ops.gemm_backward, one gradient per call) against cuDNN's convolution_backward on fp16
    channels-last (convs) or cuBLAS through torch.autograd.grad of F.linear minus its forward (Linear).
    Algorithmic FLOP: 2 M N K for each of dA and dW."""
    import torch.nn.functional as F
    if conv is not None:
        nb, hh, ww = conv
        c = k // 9
        m = nb * ((hh - 1) // stride + 1) * ((ww - 1) // stride + 1)
        a, kw = h(nb * hh * ww, c), dict(conv=(nb, hh, ww, c), conv_stride=stride)
        tag = f"conv{stride} B={nb} {hh}x{ww} {c}->{n}"
    else:
        a, kw = h(m, k), {}
        tag = f"linear m={m} n={n} k={k}"
    w, dd = h(n, k), h(m, n)
    fl = 2.0 * m * n * k
    da = torch.empty(a.shape, dtype=torch.float16, device=D)
    dw = torch.empty(n, k, device=D)
    db = torch.empty(n, device=D)
    timeit(f"ours dA    {tag}", lambda: ops.gemm_backward(a, w, dd, grads=("a",), out_da=da, **kw), flops=fl)
    timeit(f"ours dW    {tag}", lambda: ops.gemm_backward(a, w, dd, grads=("b",), out_db=dw, **kw), flops=fl)
    timeit(f"ours dbias {tag}", lambda: ops.gemm_backward(a, w, dd, grads=("bias",), out_dbias=db, **kw),
           bytes_=2.0 * m * n)
    if conv is not None:
        x = a.view(nb, hh, ww, c).permute(0, 3, 1, 2)  # NCHW view of NHWC memory: channels-last
        wt = w.view(n, 3, 3, c).permute(0, 3, 1, 2)
        g = dd.view(nb, -1, n).view(nb, (hh - 1) // stride + 1, (ww - 1) // stride + 1, n).permute(0, 3, 1, 2)
        cb = lambda mask: torch.ops.aten.convolution_backward(g, x, wt, [n], [stride] * 2, [1, 1], [1, 1], False,
                                                              [0, 0], 1, mask)
        timeit_eager(f"cudnn dA   {tag}", lambda: cb([True, False, False]), flops=fl)
        timeit_eager(f"cudnn dW   {tag}", lambda: cb([False, True, False]), flops=fl)
    else:
        at, wt = a.clone().requires_grad_(), w.clone().requires_grad_()
        with torch.no_grad():
            timeit_eager(f"cublas fwd        {tag}", lambda: F.linear(a, w), flops=fl)
        timeit_eager(f"cublas fwd+dA+dW  {tag} (subtract fwd)",
                     lambda: torch.autograd.grad(F.linear(at, wt), (at, wt), dd), flops=3 * fl)


def norm_bwd_cases():
    """our GroupNorm(+SiLU) / LayerNorm / GEGLU backward against torch's own backward kernels on the same fp16 tensors
    (torch.autograd.grad through a recorded forward, so only the backward runs).  Bytes are computed from shapes:
    GroupNorm reads x in the statistics pass and x + dy in each of its two data passes and writes dx (12 bytes per
    element); LayerNorm reads x + dy once and writes dx (6); GEGLU reads h and dout and writes dh (10 per output)."""
    import torch.nn.functional as F
    b = 4  # BASELINE config 5: 4 samples at latent 64x64
    for hw, c1, c2 in ((4096, 320, 0), (4096, 320, 320), (4096, 640, 320), (1024, 640, 0), (1024, 1280, 640),
                       (256, 1280, 0), (256, 1280, 1280), (64, 1280, 1280)):
        c, e = c1 + c2, b * hw * (c1 + c2)
        x1, x2 = h(b * hw, c1), (h(b * hw, c2) if c2 else None)
        g_, b_, dy = f(c), f(c), h(b * hw, c)
        tag = f"B={b} hw={hw} c={c1}+{c2}"
        kw = dict(batch=b, hw=hw, eps=1e-5, silu=True, x2=x2)
        timeit(f"ours  groupnorm+silu bwd dx       {tag}",
               lambda: ops.groupnorm_backward(x1, g_, b_, dy, grads=("x",), **kw), bytes_=12.0 * e)
        timeit(f"ours  groupnorm+silu bwd dx,dg,db {tag}",
               lambda: ops.groupnorm_backward(x1, g_, b_, dy, **kw), bytes_=12.0 * e)
        xt = (torch.cat([x1, x2], 1) if c2 else x1).view(b, hw, c).permute(0, 2, 1).detach().requires_grad_()
        gt, bt = g_.half().requires_grad_(), b_.half().requires_grad_()
        y = F.silu(F.group_norm(xt, 32, gt, bt, 1e-5))
        dyt = dy.view(b, hw, c).permute(0, 2, 1)
        timeit_eager(f"torch groupnorm+silu bwd dx,dg,db {tag}",
                     lambda: torch.autograd.grad(y, (xt, gt, bt), dyt, retain_graph=True))
    for rows, c in ((16384, 320), (4096, 640), (1024, 1280)):
        x, g_, dy = h(rows, c), f(c), h(rows, c)
        timeit(f"ours  layernorm bwd dx       rows={rows} c={c}",
               lambda: ops.layernorm_backward(x, g_, dy, grads=("x",)), bytes_=6.0 * rows * c)
        timeit(f"ours  layernorm bwd dx,dg,db rows={rows} c={c}", lambda: ops.layernorm_backward(x, g_, dy),
               bytes_=6.0 * rows * c)
        xt, gt, bt = x.clone().requires_grad_(), g_.half().requires_grad_(), f(c).half().requires_grad_()
        y = F.layer_norm(xt, (c,), gt, bt, 1e-5)
        timeit_eager(f"torch layernorm bwd dx,dg,db rows={rows} c={c}",
                     lambda: torch.autograd.grad(y, (xt, gt, bt), dy, retain_graph=True))
    for m, n in ((16384, 1280), (4096, 2560), (1024, 5120)):
        hh, dout = h(m, 2 * n), h(m, n)
        timeit(f"ours  geglu fwd m={m} n={n}", lambda: ops.geglu(hh), bytes_=6.0 * m * n)
        timeit(f"ours  geglu bwd m={m} n={n}", lambda: ops.geglu_backward(hh, dout), bytes_=10.0 * m * n)
        ht = hh.clone().requires_grad_()
        v, g = ht.chunk(2, dim=-1)
        y = v * F.gelu(g)
        timeit_eager(f"torch geglu bwd m={m} n={n}", lambda: torch.autograd.grad(y, ht, dout, retain_graph=True),
                     bytes_=10.0 * m * n)


def direct_bwd_cases():
    """our direct-conv backward against cuDNN's convolution_backward (fp16, channels-last) on the same tensors, our
    skinny-Linear backward against torch's fp32 matmuls, and our upsample backward, at the training shapes (4 samples,
    512^2 pose maps, 64^2 latent).  Conv FLOP are algorithmic (2 M N K per gradient); the SiLU rows include the
    recomputed forward.  Skinny bytes: W read once (fp16) plus dW written (fp32); upsample: dy read + dx written."""
    from tests.direct_bwd_cases import HINT_LAYERS
    b, s = 4, 512
    convs = [(cin, cout, st, s // div, True) for cin, cout, st, div in HINT_LAYERS] + [(4, 320, 1, 64, False),
                                                                                        (320, 4, 1, 64, False)]
    for cin, cout, st, hw, silu in convs:
        ho = (hw - 1) // st + 1
        x, wt, dy, bias = h(b * hw * hw, cin), h(cout, 9 * cin) * 0.1, h(b * ho * ho, cout), f(cout)
        fl = 2.0 * b * ho * ho * cout * 9 * cin
        tag = f"B={b} {hw}x{hw} {cin}->{cout} s{st}"
        kw = dict(batch=b, h=hw, w=hw, cin=cin, cout=cout, stride=st, bias=bias)
        wt_t = ops.flip_conv_weight(wt, cin=cin, cout=cout)
        dw, db = torch.empty(cout, cin, 3, 3, device=D), torch.empty(cout, device=D)
        dx = torch.empty(b * hw * hw, cin, dtype=torch.float16, device=D)
        if cin != 3:
            timeit(f"ours  dx      {tag}", lambda: ops.conv3x3_direct_backward(x, wt, dy, grads=("x",), wt_t=wt_t,
                                                                                out_dx=dx, **kw), flops=fl)
        timeit(f"ours  dW,db   {tag}", lambda: ops.conv3x3_direct_backward(x, wt, dy, grads=("w", "bias"), out_dw=dw,
                                                                            out_dbias=db, **kw), flops=fl)
        grads = ("w", "bias") if cin == 3 else ("x", "w", "bias")
        timeit(f"ours  all{'+silu' if silu else '     '} {tag}",
               lambda: ops.conv3x3_direct_backward(x, wt, dy, grads=grads, wt_t=wt_t, silu=silu, out_dx=dx,
                                                   out_dw=dw, out_dbias=db, **kw), flops=fl * len(grads[:2]))
        xc = x.view(b, hw, hw, cin).permute(0, 3, 1, 2)  # NCHW views of NHWC memory: channels-last
        wc = wt.view(cout, 3, 3, cin).permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)
        g = dy.view(b, ho, ho, cout).permute(0, 3, 1, 2)
        cb = lambda mask: torch.ops.aten.convolution_backward(g, xc, wc, [cout], [st] * 2, [1, 1], [1, 1], False,
                                                              [0, 0], 1, mask)
        if cin != 3:
            timeit_eager(f"cudnn dx      {tag}", lambda: cb([True, False, False]), flops=fl)
        timeit_eager(f"cudnn dW,db   {tag}", lambda: cb([False, True, True]), flops=fl)
        timeit_eager(f"cudnn all     {tag}", lambda: cb([cin != 3, True, True]), flops=fl * len(grads[:2]))
    for rows, n, k, silu in ((4, 20160, 1280, True), (4, 9600, 1280, True), (4, 1280, 320, False),
                             (4, 1280, 1280, True)):
        x, w, dy = f(rows, k), h(n, k) * 0.03, f(rows, n)
        dx, dw, db = torch.empty(rows, k, device=D), torch.empty(n, k, device=D), torch.empty(n, device=D)
        tag = f"rows={rows} n={n} k={k}"
        timeit(f"ours  skinny dx,dW,db {tag}",
               lambda: ops.skinny_linear_backward(x, w, dy, silu_in=silu, out_dx=dx, out_dw=dw, out_dbias=db),
               bytes_=6.0 * n * k)
        w32 = w.float()
        timeit_eager(f"torch linear dx,dW,db (fp32 mm) {tag}", lambda: (dy @ w32, dy.t() @ x, dy.sum(0)),
                     bytes_=8.0 * n * k)
    for hw, c in ((8, 1280), (16, 1280), (32, 640)):
        dy = h(b * 4 * hw * hw, c)
        e = b * hw * hw * c
        timeit(f"ours  upsample2x bwd B={b} {hw}x{hw}->{2 * hw} c={c}",
               lambda: ops.upsample2x_backward(dy, batch=b, h=hw, w=hw, c=c), bytes_=10.0 * e)
        dyt = dy.view(b, 2 * hw, 2 * hw, c).permute(0, 3, 1, 2)
        timeit_eager(f"torch upsample_nearest2d bwd B={b} {hw}x{hw}->{2 * hw} c={c}",
                     lambda: torch.ops.aten.upsample_nearest2d_backward(dyt, [2 * hw, 2 * hw], [b, c, hw, hw]),
                     bytes_=10.0 * e)


def igemm_case(b, hh, ww, cin, cout, stride=1):
    """one 3x3 conv (+ bias) four ways: TMA im2col loads, im2col3x3 + GEMM, the TMA-box path where the pixels tile,
    and cuDNN (fp16 channels-last F.conv2d)"""
    from magicdance_b200.engine import _igemm_ok
    x, w, bias = h(b * hh * ww, cin), h(cout, 9 * cin), f(cout)
    ho, wo = (hh - 1) // stride + 1, (ww - 1) // stride + 1
    fl = 2.0 * b * ho * wo * cout * 9 * cin
    conv = (b, hh, ww, cin)
    tag = f"B={b} {hh}x{ww} {cin}->{cout} s={stride}"
    timeit(f"im2col-mode TMA  {tag}", lambda: ops.conv3x3_igemm(x, w, conv=conv, conv_stride=stride, bias=bias),
           flops=fl)
    timeit(f"im2col3x3+gemm   {tag}", lambda: ops.gemm(ops.im2col3x3(x, batch=b, h=hh, w=ww, c=cin, stride=stride), w,
                                                        bias=bias), flops=fl)
    if _igemm_ok(ho, wo, cin):
        timeit(f"box TMA          {tag}", lambda: ops.gemm(x, w, bias=bias, conv=conv, conv_stride=stride), flops=fl)
    xc = x.reshape(b, hh, ww, cin).permute(0, 3, 1, 2)
    wc = w.reshape(cout, 3, 3, cin).permute(0, 3, 1, 2)
    bh = bias.half()
    timeit(f"cuDNN            {tag}", lambda: torch.nn.functional.conv2d(xc, wc, bh, padding=1, stride=stride),
           flops=fl)


SKINNY_PLANS = (("compute-bound plan", dict(skinny_ctas=0)), ("skinny plan (<= 96 CTAs)", {}),
                 ("skinny, <= 132 CTAs", dict(skinny_ctas=132)), ("skinny, >= 4 chunks/split", dict(split_min_chunks=4)))


def skinny_cases():
    """The weight-bound layers of a one-frame step (the UNet pair at M = 2hw, the pose net at M = hw), each under the
    plans of SKINNY_PLANS, alternated twice in this process.  Every one of the `reps` launches reads its own copy of the
    weights, so they come from HBM (not from an L2 warmed by the previous launch); GB/s = weight bytes / time."""
    reps = 20
    cases = []
    for m in (128, 64):  # 8x8: encoder 10-11, middle, decoder 0-2
        cases += [(f"8x8 M={m} proj/to_out 1280x1280", m, 1280, 1280, None),
                  (f"8x8 M={m} attn1 q|k 2560x1280", m, 2560, 1280, None),
                  (f"8x8 M={m} ff out 1280x5120", m, 1280, 5120, None),
                  (f"8x8 M={m} skip 1x1 1280x2560", m, 1280, 2560, None),
                  (f"8x8 M={m} conv 1280->1280", m, 1280, 9 * 1280, (m // 64, 8, 8, 1280)),
                  (f"8x8 M={m} conv 2560->1280", m, 1280, 9 * 2560, (m // 64, 8, 8, 2560))]
    cases += [("8x8 attn1 V^T M=1280 N=128", 1280, 128, 1280, None),
              ("16x16 M=512 1280x1280", 512, 1280, 1280, None), ("16x16 M=256 1280x1280", 256, 1280, 1280, None),
              ("16x16 M=512 conv 1280->1280", 512, 1280, 9 * 1280, (2, 16, 16, 1280)),
              ("14x8 B=2 conv 1280->1280 (im2col)", 224, 1280, 9 * 1280, (2, 14, 8, 1280))]
    for name, m, n, k, conv in cases:
        a = h(m, k) if conv is None else h(conv[0] * conv[1] * conv[2], conv[3])
        ws = [h(n, k) for _ in range(reps)]
        bias, out = f(n), torch.empty(m, n, device=D, dtype=torch.float16)
        if conv is None:
            run = lambda w: ops.gemm(a, w, bias=bias, out=out)
        elif conv[1:3] == (14, 8):
            run = lambda w: ops.conv3x3_igemm(a, w, conv=conv, bias=bias, out=out)
        else:
            run = lambda w: ops.gemm(a, w, bias=bias, conv=conv, out=out)
        res = {}
        for _ in range(2):
            for label, kw in SKINNY_PLANS:
                with ops.tuning(**kw):
                    run(ws[0])
                    torch.cuda.synchronize()
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g):
                        for w in ws:
                            run(w)
                for _ in range(3):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    g.replay()
                    e1.record()
                    torch.cuda.synchronize()
                    us = e0.elapsed_time(e1) * 1e3 / reps
                    res[label] = min(res.get(label, 1e9), us)
                del g
        for label, _ in SKINNY_PLANS:
            us = res[label]
            print(f"{name:36s} {label:28s} {us:8.2f} us  {2.0 * n * k / us / 1e3:7.1f} GB/s", flush=True)


def main():
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    ops.ensure_device()
    if which == "skinny":
        import subprocess
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip()
        print(f"GPU: {torch.cuda.get_device_name()} | nvidia-smi: {smi}", flush=True)
        skinny_cases()
        return
    if which == "igemm":
        import subprocess
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip()
        print(f"GPU: {torch.cuda.get_device_name()} | nvidia-smi: {smi}", flush=True)
        # the UNet's 3x3 convs at a 112x64 latent (512x896 portrait), B = 2 (one CFG pair), and a box size for scale
        for hh, ww, cin, cout in ((112, 64, 320, 320), (28, 16, 640, 640), (14, 8, 1280, 1280), (14, 8, 2560, 1280),
                                  (56, 32, 960, 320), (64, 64, 320, 320)):
            igemm_case(2, hh, ww, cin, cout)
        for hh, ww, c in ((112, 64, 320), (28, 16, 640)):
            igemm_case(2, hh, ww, c, c, stride=2)
        return
    if which == "direct_bwd":
        import subprocess
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip()
        print(f"GPU: {torch.cuda.get_device_name()} | nvidia-smi: {smi}", flush=True)
        direct_bwd_cases()
        return
    if which == "norm_bwd":
        import subprocess
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip()
        print(f"GPU: {torch.cuda.get_device_name()} | nvidia-smi: {smi}", flush=True)
        norm_bwd_cases()
        return
    if which == "gemm_bwd":
        import subprocess
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip()
        print(f"GPU: {torch.cuda.get_device_name()} | nvidia-smi: {smi}", flush=True)
        # BASELINE config 5: 4 samples at latent 64x64 (16384 tokens); the UNet's Linear and 3x3 conv shapes
        for m, n, k in ((16384, 320, 320), (16384, 2560, 320), (16384, 320, 1280), (1024, 1280, 1280), (308, 320, 768)):
            gemm_bwd_case(m, n, k)
        for hw, cin, cout in ((64, 320, 320), (32, 640, 640), (16, 1280, 1280), (8, 1280, 1280), (8, 2560, 1280),
                              (64, 960, 320)):
            gemm_bwd_case(0, cout, 9 * cin, conv=(4, hw, hw))
        for hw, c in ((64, 320), (32, 640), (16, 1280)):
            gemm_bwd_case(0, c, 9 * c, conv=(4, hw, hw), stride=2)
        return
    if which == "attn_bwd":
        import subprocess
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip()
        print(f"GPU: {torch.cuda.get_device_name()} | nvidia-smi: {smi}", flush=True)
        # BASELINE config 5: 4 samples at latent 64x64, 8 heads; self + bank at every level, the text source at 64x64
        attn_bwd_case(4, 40, 4096, 4096, 4096)
        attn_bwd_case(4, 80, 1024, 1024, 1024)
        attn_bwd_case(4, 160, 256, 256, 256)
        attn_bwd_case(4, 160, 64, 64, 64)
        attn_bwd_case(4, 40, 4096, 77)
        return
    if which in ("all", "gemm"):
        for m, n, k in ((128, 160, 64), (128, 160, 640), (128, 160, 2560), (128, 1280, 1280)):
            gemm_case(m, n, k, res=False, bias=False)
        for s in (1, 2):
            gemm_case(4096, 320, 320, s)
        for s in (1, 2, 4):
            gemm_case(1024, 640, 640, s)
        for s in (1, 5, 10):
            gemm_case(256, 1280, 1280, s)
        for s in (1, 4, 8, 16):
            gemm_case(64, 1280, 1280, s)
        gemm_case(4096, 320, 1280)
        gemm_case(8192, 320, 320)
        gemm_case(32768, 320, 320)
        x, (wp, bp) = h(4096, 320), pack_geglu(torch.randn(2560, 320), torch.randn(2560), D)
        timeit("geglu m=4096 c=320", lambda: ops.gemm(x, wp, bias=bp, epilogue=ops.EPI_GEGLU), flops=2.0 * 4096 * 2560 * 320)
    if which in ("all", "conv"):
        for s in (1, 2, 4):
            conv_case(1, 64, 64, 320, 320, s)
        conv_case(8, 64, 64, 320, 320)
        conv_case(1, 64, 64, 640, 320, 2)
        for s in (1, 2, 4):
            conv_case(1, 32, 32, 640, 640, s)
        conv_case(8, 32, 32, 640, 640)
        for s in (1, 4, 9):
            conv_case(1, 16, 16, 1280, 1280, s)
        for s in (1, 8, 16):
            conv_case(1, 8, 8, 1280, 1280, s)
        conv_case(2, 8, 8, 2560, 1280, 16)
        conv_case(8, 8, 8, 1280, 1280, 4)
    if which == "pair":
        # two-CTA-per-SM 128 x BN tiles vs the one-CTA-per-SM large-grid tiles (128 x 256 / deep rings), shape by shape, at the cond+uncond batch of one frame (2) and of eight frames (16)
        big = 1 << 30
        for label, tune in (("single-CTA tiles", dict(pair_min_tiles=big)), ("pair kernel (forced)", dict(pair_min_tiles=1))):
            print(f"--- {label}", flush=True)
            with ops.tuning(**tune):
                for b in (2, 16):
                    conv_case(b, 64, 64, 320, 320)
                    conv_case(b, 64, 64, 640, 320)
                    conv_case(b, 32, 32, 640, 640)
                    conv_case(b, 32, 32, 1280, 640)
                    conv_case(b, 16, 16, 1280, 1280)
                    conv_case(b, 8, 8, 1280, 1280)
                    gemm_case(b * 4096, 320, 320)
                    gemm_case(b * 4096, 320, 1280)
                    gemm_case(b * 1024, 640, 640)
                    gemm_case(b * 1024, 640, 2560)
                    gemm_case(b * 256, 1280, 1280)
                    gemm_case(b * 256, 1280, 5120)
                    for hw, c in ((4096, 320), (1024, 640), (256, 1280)):
                        x, (wp, bp) = h(b * hw, c), pack_geglu(torch.randn(8 * c, c), torch.randn(8 * c), D)
                        timeit(f"geglu m={b * hw} c={c}", lambda: ops.gemm(x, wp, bias=bp, epilogue=ops.EPI_GEGLU),
                               flops=2.0 * b * hw * 8 * c * c)
        return
    if which == "gn":
        # GroupNorm paths by batch: mode 1 = stats (+ last-CTA fold) -> apply, mode 2 = single-launch cluster kernel
        for b in (2, 4, 8, 16, 25):
            for (hw, c1, c2) in ((4096, 320, 0), (4096, 640, 320), (1024, 640, 0), (1024, 1280, 640), (256, 1280, 0),
                                 (256, 1280, 1280), (64, 1280, 1280)):
                x1 = h(b * hw, c1)
                x2 = h(b * hw, c2) if c2 else None
                g_, b_ = f(c1 + c2), f(c1 + c2)
                for mode in (1, 2):
                    timeit(f"groupnorm B={b} hw={hw} c={c1}+{c2} mode={mode}",
                           lambda: ops.groupnorm(x1, g_, b_, batch=b, hw=hw, eps=1e-5, silu=True, x2=x2, mode=mode),
                           bytes_=3.0 * b * hw * (c1 + c2) * 2)
        return
    if which == "deepk":
        # the single-frame weight-streaming layers (cond+uncond batch of 2) with COLD weights, as inside a step (each
        # step streams 2.4 GB of weights through a 50 MB L2): eight weight copies are cycled; 80- vs 160-wide tiles
        # and the split-K factor
        def cold(name, m, n, k, conv, flops):
            ws = [h(n, k) for _ in range(max(2, int(300e6 / (2.0 * n * k)) + 1))]
            x = h(m, conv[3] if conv else k)
            bias, res = f(n), h(m, n)
            for bn_below, bnl in ((1 << 30, 80), (0, 160)):
                for sp in (1, 2, 4, 8):
                    if k // 64 < 4 * sp:
                        continue
                    state = {"i": 0}

                    def fn():
                        w = ws[state["i"] % len(ws)]
                        state["i"] += 1
                        ops.gemm(x, w, bias=bias, residual=res, splits=sp, **({"conv": conv} if conv else {}))
                    with ops.tuning(bn80_below=bn_below, pair_min_tiles=1 << 30):
                        timeit(f"{name} bn={bnl} splits={sp}", fn, reps=len(ws) * 2, flops=flops)
        for (hh, cin, cout) in ((16, 1280, 1280), (16, 2560, 1280), (8, 1280, 1280), (8, 2560, 1280), (32, 640, 640),
                                (32, 1280, 640), (64, 320, 320)):
            m = 2 * hh * hh
            cold(f"conv B=2 {hh}x{hh} {cin}->{cout}", m, cout, 9 * cin, (2, hh, hh, cin), 2.0 * m * cout * 9 * cin)
        for (m, n, k) in ((512, 1280, 5120), (512, 1280, 1280), (2048, 640, 2560), (2048, 640, 640), (8192, 320, 1280)):
            cold(f"gemm m={m} n={n} k={k}", m, n, k, None, 2.0 * m * n * k)
        return
    if which in ("all", "attn"):
        # d=40 (the 64x64 level, self tokens + bank): the register-capped two-CTA-per-SM variant (key 0) against the
        # one-CTA-per-SM variant (key 2^30) at the cond|uncond batch of one frame (512 CTAs) and of eight (4096 CTAs)
        for b in (2, 16):
            for key in (0, 1 << 30):
                with ops.tuning(attn40_2q_min_ctas=key):
                    print(f"attn40_2q_min_ctas={key}:", end=" ", flush=True)
                    attn_case(b, 40, 4096, 4096, 4096)
        attn_case(1, 40, 4096, 77)
        attn_case(16, 80, 1024, 1024, 1024)
        attn_case(1, 80, 1024, 1024, 1024)
        attn_case(1, 80, 1024, 77)
        attn_case(1, 160, 256, 256, 256)
        attn_case(1, 160, 64, 64, 64)
        attn_case(1, 160, 256, 77)
    if which in ("all", "misc"):
        for (b, hw, c1, c2) in ((1, 4096, 320, 0), (1, 4096, 640, 320), (1, 1024, 640, 0), (1, 256, 1280, 1280), (1, 64, 1280, 1280), (8, 4096, 320, 0)):
            x1 = h(b * hw, c1)
            x2 = h(b * hw, c2) if c2 else None
            g_, b_ = f(c1 + c2), f(c1 + c2)
            timeit(f"groupnorm B={b} hw={hw} c={c1}+{c2}", lambda: ops.groupnorm(x1, g_, b_, batch=b, hw=hw, eps=1e-5, silu=True, x2=x2),
                   bytes_=2.0 * b * hw * (c1 + c2) * 3)
        for rows, c in ((4096, 320), (1024, 640), (256, 1280)):
            x, g_, b_ = h(rows, c), f(c), f(c)
            timeit(f"layernorm rows={rows} c={c}", lambda: ops.layernorm(x, g_, b_), bytes_=4.0 * rows * c)
        a, b2 = h(4096, 320), h(4096, 320)
        timeit("add 4096x320", lambda: ops.add(a, b2, batch=1), bytes_=6.0 * 4096 * 320)
        x = h(1024, 640)
        timeit("upsample 32x32x640", lambda: ops.upsample2x(x, batch=1, h=32, w=32, c=640))
        x = h(4096, 320)
        timeit("im2col 64x64x320", lambda: ops.im2col3x3(x, batch=1, h=64, w=64, c=320, stride=2))
        e, w, bb = f(1, 1280), h(20160, 1280), f(20160)
        timeit("skinny_linear 1x20160x1280", lambda: ops.skinny_linear(e, w, bb, silu_in=True), bytes_=2.0 * 20160 * 1280)
        for (hh, cin, cout, s) in ((512, 3, 16, 1), (512, 16, 16, 1), (512, 16, 32, 2), (256, 32, 32, 1), (256, 32, 96, 2),
                                   (128, 96, 96, 1), (128, 96, 256, 2)):
            x, w, bb = h(hh * hh, cin), h(cout, 9 * cin), f(cout)
            ho = (hh - 1) // s + 1
            timeit(f"direct conv {hh}x{hh} {cin}->{cout} s={s}",
                   lambda: ops.conv3x3_direct(x, w, bb, batch=1, h=hh, w=hh, cin=cin, cout=cout, stride=s, silu=True),
                   reps=5, flops=2.0 * ho * ho * cout * 9 * cin)
        x = h(4096, 4)
        w, bb = h(320, 36), f(320)
        timeit("direct conv_in 64x64 4->320", lambda: ops.conv3x3_direct(x, w, bb, batch=1, h=64, w=64, cin=4, cout=320))
        x = h(4096, 320)
        w, bb = h(4, 2880), f(4)
        timeit("direct conv_out 64x64 320->4", lambda: ops.conv3x3_direct(x, w, bb, batch=1, h=64, w=64, cin=320, cout=4))


if __name__ == "__main__":
    main()
