"""Torch-tensor front end of the C ABI (include/magicdance_b200.h).

PyTorch is plumbing here: it owns device memory and the current CUDA stream; every function
below launches OUR kernels through ctypes.  No function has a PyTorch/CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import math
import os

import torch

from . import _lib

EPI_NONE, EPI_GEGLU = 0, 1
SKINNY_MAX_ROWS = 16  # mdb_skinny_linear_f32: rows per launch
_GEMM_DEBUG = os.environ.get("MDB_GEMM_DEBUG", "0") == "1"
TRACE = None  # set to a list to record (m, n, k, conv, epilogue, splits, k2) of every gemm() call (bench.py)


class tuning:
    """`with ops.tuning(pair_min_tiles=1):` — the library's launch heuristics (include/magicdance_b200.h
    mdb_set_tuning) for the duration of the block; tests use it to force a kernel variant onto small problems.
    Launches captured into CUDA graphs keep the variant they were captured with."""
    _KEYS = {"pair_min_tiles": _lib.TUNE_GEMM_PAIR_MIN_TILES,
             "attn40_2q_min_ctas": _lib.TUNE_ATTN40_2Q_MIN_CTAS, "bn80_below": _lib.TUNE_GEMM_BN80_BELOW,
             "skinny_ctas": _lib.TUNE_GEMM_SKINNY_CTAS, "split_min_chunks": _lib.TUNE_GEMM_SPLIT_MIN_CHUNKS}

    def __init__(self, **kw):
        self.want = {self._KEYS[k]: int(v) for k, v in kw.items() if v is not None}

    def __enter__(self):
        lib = _lib.load()
        self.old = {k: int(lib.mdb_get_tuning(k)) for k in self.want}
        for k, v in self.want.items():
            _lib.check(lib.mdb_set_tuning(k, v), "set_tuning")
        return self

    def __exit__(self, *a):
        lib = _lib.load()
        for k, v in self.old.items():
            lib.mdb_set_tuning(k, v)


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return None if t is None else t.data_ptr()


def _chk(t: torch.Tensor, dtype, name):
    if not t.is_cuda:
        raise RuntimeError(f"magicdance_b200: {name} must be a CUDA tensor (no CPU fallback exists for the hot path)")
    if t.dtype != dtype:
        raise RuntimeError(f"magicdance_b200: {name} must be {dtype}, got {t.dtype}")


def require_cuda(device):
    """The single place that decides where the networks may live: an sm_90 CUDA device, nothing else."""
    if torch.device(device).type != "cuda":
        raise RuntimeError("magicdance_b200: the networks run only on an sm_90 CUDA device — move the model to "
                           "the GPU first (there is no CPU/PyTorch fallback for the hot path)")


def ensure_device():
    lib = _lib.load()
    if not torch.cuda.is_available():
        raise RuntimeError("magicdance_b200: no CUDA device visible; the hot path has no CPU fallback")
    _lib.check(lib.mdb_device_check(), "device_check")
    return lib


def launch_count() -> int:
    return int(_lib.load().mdb_launch_count())


_ws_cache = {}


_ws_tag = 0  # scratch buffers are per "lane": concurrent streams must not share split-K / GroupNorm scratch


class workspace_lane:
    """`with ops.workspace_lane(1):` — kernels issued inside use their own scratch buffers, so a second
    CUDA stream can run another branch of the step concurrently (pipeline.GraphedDenoiser)."""

    def __init__(self, tag):
        self.tag = tag

    def __enter__(self):
        global _ws_tag
        self.prev, _ws_tag = _ws_tag, self.tag

    def __exit__(self, *a):
        global _ws_tag
        _ws_tag = self.prev


def current_lane():
    return _ws_tag


_ws_retired = []  # outgrown buffers stay alive: captured CUDA graphs hold raw pointers into them


def _workspace(key, numel, dtype, device, zero=False):
    """Per-(key, device, lane) scratch buffer, grown geometrically.  A buffer that is outgrown is RETIRED, never
    freed: launches captured into CUDA graphs keep its address, and a replay must not touch memory the caching
    allocator has handed to somebody else."""
    k = (key, device, _ws_tag)
    t = _ws_cache.get(k)
    if t is None or t.numel() < numel or t.dtype != dtype:
        if t is not None:
            _ws_retired.append(t)
            numel = max(numel, 2 * t.numel())
        alloc = torch.zeros if zero else torch.empty
        t = alloc(max(numel, 1), dtype=dtype, device=device)
        _ws_cache[k] = t
    return t


def _gemm_m(a, conv, conv_stride, m):
    """rows of D: the output pixels of the 3x3 pad-1 conv, else m (default: a's rows)"""
    if conv is not None:
        nb, h, wd, _ = conv
        return nb * ((h - 1) // conv_stride + 1) * ((wd - 1) // conv_stride + 1)
    return a.shape[0] if m is None else m


def _fill_fwd_desc(g, a, w, a2, conv, conv_stride, m):
    """fills the A-side fields (a, a2, conv geometry) and m, n, k of the forward GemmDesc g; returns (m, k1)"""
    n, k = w.shape
    if conv is not None:
        nb, h, wd, c = conv
        assert conv_stride in (1, 2) and a.is_contiguous() and a.numel() == nb * h * wd * c
        g.conv, g.nb, g.h, g.w, g.c = conv_stride, nb, h, wd, c  # descriptor: conv = 1 (stride 1) | 2 (stride 2)
        g.a, g.lda, g.k1 = a.data_ptr(), c, k
    else:
        assert a.dim() == 2 and a.stride(1) == 1
        g.a, g.lda, g.k1 = a.data_ptr(), a.stride(0), a.shape[1]
        if a2 is not None:
            _chk(a2, torch.float16, "a2")
            assert a2.dim() == 2 and a2.stride(1) == 1 and a2.shape[0] == a.shape[0]
            g.a2, g.lda2 = a2.data_ptr(), a2.stride(0)
            assert a.shape[1] + a2.shape[1] == k
        else:
            assert a.shape[1] == k, (a.shape, w.shape)
    m = _gemm_m(a, conv, conv_stride, m)
    g.m, g.n, g.k = m, n, k
    return m, g.k1


def _fill_epilogue(g, w, out, n_out, device, bias, bias_batch_stride, rows_per_batch, residual, splits):
    """fills the B operand and the epilogue fields (out, bias or per-batch bias, residual, split count and split-K
    workspace) of the forward GemmDesc g whose A side is filled; returns out, a new [m, n_out] tensor when None"""
    m = g.m
    if out is None:
        out = torch.empty((m, n_out), dtype=torch.float16, device=device)
    _chk(out, torch.float16, "out")
    assert out.dim() == 2 and out.stride(1) == 1 and out.shape[0] >= m and out.shape[1] == n_out, (out.shape, m, n_out)
    assert w.stride(1) == 1
    g.b, g.ldb = w.data_ptr(), w.stride(0)
    g.d, g.ldd = out.data_ptr(), out.stride(0)
    if bias is not None:
        _chk(bias, torch.float32, "bias")
        g.bias, g.bias_batch_stride, g.rows_per_batch = bias.data_ptr(), bias_batch_stride, rows_per_batch
    if residual is not None:
        _chk(residual, torch.float16, "residual")
        assert residual.dim() == 2 and residual.stride(1) == 1
        g.residual, g.ldr = residual.data_ptr(), residual.stride(0)
    g.splits = splits
    if splits > 8:
        # the library rounds the count so that no split is empty (12 splits of 20 K chunks run as 10); up to 8 splits
        # reduce inside a cluster, more through this workspace
        g.splitk_ws = _workspace("splitk", splits * m * g.n, torch.float32, device).data_ptr()
    return out


def gemm(a, w, *, out=None, bias=None, bias_batch_stride=0, rows_per_batch=0, residual=None, epilogue=EPI_NONE,
         a2=None, conv=None, conv_stride=1, splits=0, m=None, ln_u=None, ln_eps=1e-5):
    """D = epilogue(A @ W^T).  a: [M, K1] fp16 (last dim contiguous, row stride arbitrary) or, with
    conv=(nb, h, w, c), an NHWC activation; w: [N, K] fp16; a2: optional second K-range source.
    splits: 0 = the library picks tile width and split-K (1 ... 8, reduced inside a thread-block cluster),
    1 = no split, n = at most n splits (no split is left empty; a count above 8 goes through an fp32 workspace).
    ln_u: LayerNorm over a's rows folded into the GEMM — w must be W diag(gamma), bias W beta (+ b), ln_u the row sums
    of w (engine.fold_layernorm); D = rstd_r (a w^T - mean_r ln_u) + bias.  Small grids only."""
    lib = _lib.load()
    _chk(a, torch.float16, "a")
    _chk(w, torch.float16, "w")
    g = _lib.GemmDesc()
    n, k = w.shape
    m, _ = _fill_fwd_desc(g, a, w, a2, conv, conv_stride, m)
    out = _fill_epilogue(g, w, out, n // 2 if epilogue == EPI_GEGLU else n, a.device, bias, bias_batch_stride,
                         rows_per_batch, residual, 1 if ln_u is not None else splits)  # the folded LayerNorm: no split
    g.epilogue = epilogue
    if ln_u is not None:
        _chk(ln_u, torch.float32, "ln_u")
        assert conv is None and a2 is None and ln_u.numel() == n and ln_u.is_contiguous()
        g.ln_u, g.ln_eps = ln_u.data_ptr(), float(ln_eps)
    if TRACE is not None:
        TRACE.append((m, n, k, (tuple(conv) + (conv_stride,)) if conv is not None else None, epilogue, g.splits,
                      a2.shape[1] if a2 is not None else 0))
    if _GEMM_DEBUG:  # MDB_GEMM_DEBUG=1: name every GEMM before it runs and wait for it (pins down a hanging shape)
        import sys
        print(f"gemm m={m} n={n} k={k} conv={conv} epi={epilogue} splits={g.splits} a2={a2 is not None} lda={g.lda} "
              f"ldd={g.ldd} bias={bias is not None} bbs={g.bias_batch_stride} res={residual is not None}",
              file=sys.stderr, flush=True)
    _lib.check(lib.mdb_gemm_f16(C.byref(g), _stream()), "gemm_f16")
    if _GEMM_DEBUG:
        torch.cuda.synchronize()
    return out


_DTYPES = {torch.float16: 0, torch.float32: 1}  # MDB_DTYPE_F16 / MDB_DTYPE_F32


def _dest(t, shape, dtype, device, name, *, any_float=False, contiguous=False, rows8=False, numel=False, zero=False):
    """The destination of one gradient: a new tensor of `shape` and `dtype` (zero-filled with zero) when the caller
    gave none, else the caller's out_* tensor t, checked before any kernel writes through it.  t must be of dtype
    (float16 or float32 with any_float: the gradient then takes t's dtype), dense with contiguous, else 2-D with unit
    column stride (and with rows8 a row stride that is a multiple of 8), and of `shape` (with numel: of as many
    elements, in any shape)."""
    if t is None:
        return (torch.zeros if zero else torch.empty)(shape, dtype=dtype, device=device)
    dtypes = tuple(_DTYPES) if any_float else (dtype,)
    kind = " or ".join(str(d).removeprefix("torch.") for d in dtypes)
    if contiguous:
        ok, want = t.is_contiguous(), f"a contiguous {kind} tensor"
    else:
        ok = t.dim() == 2 and t.stride(1) == 1 and (not rows8 or t.stride(0) % 8 == 0)
        want = f"a 2-D {kind} tensor with unit column stride" + (" and a row stride that is a multiple of 8" if rows8
                                                                  else "")
    if t.dtype not in dtypes or not ok:
        raise RuntimeError(f"magicdance_b200: {name} must be {want} (got {t.dtype}, strides {tuple(t.stride())})")
    if (t.numel() != math.prod(shape)) if numel else (tuple(t.shape) != tuple(shape)):
        want = f"{math.prod(shape)} elements" if numel else f"shape {tuple(shape)}"
        raise RuntimeError(f"magicdance_b200: {name} must have {want}, got {tuple(t.shape)}")
    _chk(t, t.dtype, name)
    return t


def _bwd_ws(desc, ws_floats, key, device, what, zero=False):
    """the scratch pointer of a backward descriptor: ws_floats(desc) fp32 elements of the `key` workspace (a negative
    answer is the library's argument error, raised as `what`'s)"""
    need = int(ws_floats(C.byref(desc)))
    if need < 0:
        _lib.check(need, what)
    return _workspace(key, need, torch.float32, device, zero=zero).data_ptr()


def _wanted(ctx, **inputs):
    """the `grads` names of a backward wrapper that autograd needs: each name maps to the positions of the forward's
    inputs that receive that gradient"""
    need = ctx.needs_input_grad
    return [nm for nm, pos in inputs.items() if any(need[i] for i in pos)]


def pack_conv_weight(w):
    """Conv2d weight OIHW -> the fp16 copy the kernels read: [O][kh][kw][I] as [O, kh*kw*I] (K order tap-major,
    channel-minor)"""
    return w.detach().permute(0, 2, 3, 1).reshape(w.shape[0], -1).to(torch.float16).contiguous()


def unpack_conv_weight(w, like):
    """pack_conv_weight's layout undone as a view: w [O, kh*kw*I] in the layout of `like` (a Conv2d weight OIHW; a
    matrix such as a Linear weight keeps w's own layout)"""
    if like.dim() != 4:
        return w.view(like.shape)
    o, i, kh, kw = like.shape
    return w.view(o, kh, kw, i).permute(0, 3, 1, 2)


def _route_grad(g, operand, param):
    """(operand's gradient, param's gradient) from g, the gradient in the kernel's layout: it goes to the fp32
    parameter param, in param's layout, when the fp16 operand was packed from one, else to the operand"""
    if g is None:
        return None, None
    if param is not None:
        return None, unpack_conv_weight(g, param)
    return g.view(operand.shape).to(operand.dtype), None


def _fill_gemm_grads(g, w, dd, da_shape, da2_shape, device, ws_floats, what, *, bias_batch_stride, rows_per_batch,
                     splits, db_splits, grads, da_dtype, db_dtype, out_da, out_da2, out_db, out_dbias, accumulate):
    """fills the B operand, dD, the split counts, the gradient destinations (dA, and dA2 of da2_shape unless None; dB;
    dbias) with their accumulate flags, and the workspace of the GemmBwdDesc g whose A side is filled, in
    gemm_backward()'s conventions; returns (da, da2, dw, dbias)"""
    f, m = g.fwd, g.fwd.m
    n, k = w.shape
    assert w.stride(1) == 1 and dd.shape[0] >= m and dd.shape[1] == n, (dd.shape, m, n)
    f.b, f.ldb = w.data_ptr(), w.stride(0)
    f.splits, f.bias_batch_stride, f.rows_per_batch = splits, bias_batch_stride, rows_per_batch
    g.dd, g.lddd, g.splits = dd.data_ptr(), dd.stride(0), db_splits
    acc = set(accumulate)
    da = da2 = dw = dbias = None
    if "a" in grads:
        da = _dest(out_da, da_shape, da_dtype, device, "out_da", any_float=True)
        g.da, g.ldda, g.da_dtype, g.da_accumulate = da.data_ptr(), da.stride(0), _DTYPES[da.dtype], "a" in acc
        if da2_shape is not None:
            da2 = _dest(out_da2, da2_shape, da_dtype, device, "out_da2", any_float=True)
            g.da2, g.ldda2, g.da2_dtype = da2.data_ptr(), da2.stride(0), _DTYPES[da2.dtype]
            g.da2_accumulate = "a2" in acc
    if "b" in grads:
        dw = _dest(out_db, (n, k), db_dtype, device, "out_db", any_float=True)
        g.db, g.lddb, g.db_dtype, g.db_accumulate = dw.data_ptr(), dw.stride(0), _DTYPES[dw.dtype], "b" in acc
    if "bias" in grads:
        shape = (n,) if bias_batch_stride == 0 else (-(-m // rows_per_batch), bias_batch_stride)
        dbias = _dest(out_dbias, shape, torch.float32, device, "out_dbias", contiguous=True)
        g.dbias, g.dbias_accumulate = dbias.data_ptr(), "bias" in acc
    g.ws = _bwd_ws(g, ws_floats, "gemm_bwd", device, what)
    return da, da2, dw, dbias


def gemm_backward(a, w, dd, *, a2=None, conv=None, conv_stride=1, bias_batch_stride=0, rows_per_batch=0, splits=0,
                  db_splits=0, m=None, grads=("a", "b"), da_dtype=torch.float16, db_dtype=torch.float32, out_da=None,
                  out_da2=None, out_db=None, out_dbias=None, accumulate=(), epilogue=EPI_NONE, ln_u=None):
    """Gradients of D = gemm(a, w, ...) from dd = dL/dD (fp16 [M, N], row stride a multiple of 8), csrc/gemm_bwd.cu:
    dA = dd w, dW = dd^T a, dbias = column sums of dd (per batch element: [M / rows_per_batch, bias_batch_stride]).
    a, w, a2, conv, conv_stride, bias_batch_stride, rows_per_batch and m are gemm()'s arguments; `splits` splits the
    reduction of dA (over N), `db_splits` that of dW (over M): 0 automatic, 1 none.  `grads` names the gradients to
    compute among "a" (dA, and dA2 with a2), "b" and "bias".  Each goes to its out_* tensor when given (its dtype is
    then the gradient's dtype) or to a new one of da_dtype / db_dtype (dbias: fp32); names in `accumulate` ("a",
    "a2", "b", "bias") add into the out_* tensor instead of overwriting it.  Returns (da, da2, dw, dbias), None for a
    gradient not requested.  Deterministic; GEGLU and ln_u GEMMs are rejected."""
    lib = _lib.load()
    _chk(a, torch.float16, "a")
    _chk(w, torch.float16, "w")
    _chk(dd, torch.float16, "dd")
    assert dd.dim() == 2 and dd.stride(1) == 1
    g = _lib.GemmBwdDesc()
    m, k1 = _fill_fwd_desc(g.fwd, a, w, a2, conv, conv_stride, m)
    g.fwd.epilogue = epilogue
    if ln_u is not None:
        g.fwd.ln_u = ln_u.data_ptr()
    da_shape = (conv[0] * conv[1] * conv[2], conv[3]) if conv is not None else (m, k1)
    res = _fill_gemm_grads(g, w, dd, da_shape, (m, w.shape[1] - k1) if a2 is not None else None, a.device,
                           lib.mdb_gemm_bwd_ws_floats, "gemm_bwd_f16", bias_batch_stride=bias_batch_stride,
                           rows_per_batch=rows_per_batch, splits=splits, db_splits=db_splits, grads=grads,
                           da_dtype=da_dtype, db_dtype=db_dtype, out_da=out_da, out_da2=out_da2, out_db=out_db,
                           out_dbias=out_dbias, accumulate=accumulate)
    _lib.check(lib.mdb_gemm_bwd_f16(C.byref(g), _stream()), "gemm_bwd_f16")
    return res


def _fill_igemm_desc(g, x, w, x2, conv, conv_stride):
    """the A-side fields and m, n, k of a GemmDesc for mdb_conv3x3_igemm_*: x [nb*h*w, k1] (x2 [nb*h*w, c - k1]) with
    unit channel stride, any pixel stride"""
    nb, h, wd, c = conv
    n, k = w.shape
    assert conv_stride in (1, 2) and k == 9 * c, (conv, w.shape)
    assert x.dim() == 2 and x.stride(1) == 1 and x.shape[0] == nb * h * wd, (x.shape, conv)
    g.conv, g.nb, g.h, g.w, g.c = conv_stride, nb, h, wd, c
    g.a, g.lda = x.data_ptr(), x.stride(0)
    if x2 is not None:
        _chk(x2, torch.float16, "x2")
        assert x2.dim() == 2 and x2.stride(1) == 1 and x2.shape[0] == x.shape[0] and x.shape[1] + x2.shape[1] == c
        g.a2, g.lda2, g.k1 = x2.data_ptr(), x2.stride(0), x.shape[1]
    else:
        assert x.shape[1] == c, (x.shape, conv)
        g.k1 = c
    g.m, g.n, g.k = _gemm_m(x, conv, conv_stride, None), n, k


def conv3x3_igemm(x, w, *, conv, conv_stride=1, x2=None, out=None, bias=None, bias_batch_stride=0, rows_per_batch=0,
                  residual=None, splits=0):
    """3x3 pad-1 conv of the NHWC activation x ([nb*h*w, c], conv=(nb, h, w, c)) at any size, as an implicit GEMM whose
    activation tiles come from TMA im2col loads (mdb_conv3x3_igemm_f16); w: [cout, 9c] packed [O][kh][kw][I].  x2: a
    second source for channels [x.shape[1], c) (the concat is never materialised).  bias / per-batch bias / residual /
    splits as gemm(); at the sizes gemm(conv=...) takes, the result is bit-equal to it."""
    lib = _lib.load()
    _chk(x, torch.float16, "x")
    _chk(w, torch.float16, "w")
    g = _lib.GemmDesc()
    _fill_igemm_desc(g, x, w, x2, conv, conv_stride)
    out = _fill_epilogue(g, w, out, w.shape[0], x.device, bias, bias_batch_stride, rows_per_batch, residual, splits)
    _lib.check(lib.mdb_conv3x3_igemm_f16(C.byref(g), _stream()), "conv3x3_igemm_f16")
    return out


def conv3x3_igemm_backward(x, w, dd, *, conv, conv_stride=1, x2=None, bias_batch_stride=0, rows_per_batch=0,
                           splits=0, db_splits=0, grads=("a", "b"), da_dtype=torch.float16, db_dtype=torch.float32,
                           out_da=None, out_da2=None, out_db=None, out_dbias=None, accumulate=()):
    """Gradients of conv3x3_igemm (mdb_conv3x3_igemm_bwd_f16), in gemm_backward()'s conventions: returns (dx, dx2, dw,
    dbias); dx is [nb*h*w, x.shape[1]], dx2 the x2 channels', dw [cout, 9c] ([O][kh][kw][I]).  Deterministic."""
    lib = _lib.load()
    _chk(x, torch.float16, "x")
    _chk(w, torch.float16, "w")
    _chk(dd, torch.float16, "dd")
    assert dd.dim() == 2 and dd.stride(1) == 1
    g = _lib.GemmBwdDesc()
    _fill_igemm_desc(g.fwd, x, w, x2, conv, conv_stride)
    res = _fill_gemm_grads(g, w, dd, tuple(x.shape), tuple(x2.shape) if x2 is not None else None, x.device,
                           lib.mdb_conv3x3_igemm_bwd_ws_floats, "conv3x3_igemm_bwd_f16",
                           bias_batch_stride=bias_batch_stride, rows_per_batch=rows_per_batch, splits=splits,
                           db_splits=db_splits, grads=grads, da_dtype=da_dtype, db_dtype=db_dtype, out_da=out_da,
                           out_da2=out_da2, out_db=out_db, out_dbias=out_dbias, accumulate=accumulate)
    _lib.check(lib.mdb_conv3x3_igemm_bwd_f16(C.byref(g), _stream()), "conv3x3_igemm_bwd_f16")
    return res


class Conv3x3Igemm(torch.autograd.Function):
    """conv3x3_igemm() as an autograd op, in TcGemm's conventions: w is an fp16 activation-like operand or the packed
    fp16 copy of the fp32 OIHW parameter w_param (which then receives the fp32 gradient); the bias gets its fp32
    gradient, the residual dD.  Positional arguments in conv3x3_igemm_ad()'s order."""

    @staticmethod
    def forward(ctx, x, w, w_param, bias, residual, x2, bias_batch_stride, rows_per_batch, conv, conv_stride, splits):
        n = w.shape[0]
        m = _gemm_m(x, conv, conv_stride, None)
        out = torch.empty((m, (n + 7) // 8 * 8), dtype=torch.float16, device=x.device)[:, :n]
        conv3x3_igemm(x, w, conv=conv, conv_stride=conv_stride, x2=x2, out=out, bias=bias,
                      bias_batch_stride=bias_batch_stride, rows_per_batch=rows_per_batch, residual=residual,
                      splits=splits)
        ctx.save_for_backward(x, w, w_param, x2)
        ctx.kw = dict(conv=conv, conv_stride=conv_stride, bias_batch_stride=bias_batch_stride,
                      rows_per_batch=rows_per_batch)
        ctx.bias_shape = None if bias is None else bias.shape
        ctx.has_residual = residual is not None
        return out

    @staticmethod
    def backward(ctx, dout):
        x, w, w_param, x2 = ctx.saved_tensors
        dd = _rows8(dout)
        grads = _wanted(ctx, a=(0, 5), b=(1, 2), bias=(3,))
        dx, dx2, dw, dbias = conv3x3_igemm_backward(
            x, w, dd, x2=x2, grads=grads, db_dtype=torch.float32 if w_param is not None else torch.float16, **ctx.kw)
        g_w, g_wp = _route_grad(dw, w, w_param)
        g_bias = dbias.view(ctx.bias_shape) if dbias is not None else None
        g_res = dout if ctx.has_residual else None
        return dx, g_w, g_wp, g_bias, g_res, dx2, None, None, None, None, None


def conv3x3_igemm_ad(x, w, *, w_param=None, bias=None, bias_batch_stride=0, rows_per_batch=0, residual=None, x2=None,
                     conv, conv_stride=1, splits=0):
    """Differentiable conv3x3_igemm() (Conv3x3Igemm): the training forward's 3x3 conv at latent sizes whose pixels do
    not tile into the box path's 128-pixel TMA boxes"""
    return Conv3x3Igemm.apply(x, w, w_param, bias, residual, x2, bias_batch_stride, rows_per_batch, conv, conv_stride,
                              splits)


def pad_tokens(x, b):
    """[b*n, C] token matrix -> ([b*ldv, C], ldv) with ldv = n rounded up to a multiple of 8: zero rows after each
    sample's tokens, so that the swapped-operand GEMM W_v x^T yields V^T [C, b*ldv] whose per-sample column blocks are
    16-byte aligned (the attention kernels' ldv*_batch).  The kernels never read the padding columns: the V^T tensor
    map ends each sample at n.  x itself when n % 8 == 0 (no copy, no launch); differentiable."""
    n = x.shape[0] // b
    ldv = (n + 7) // 8 * 8
    if ldv == n:
        return x, ldv
    return torch.nn.functional.pad(x.reshape(b, n, x.shape[1]), (0, 0, 0, ldv - n)).reshape(b * ldv, -1), ldv


def _rows8(t):
    """t as a [rows, cols] fp16 matrix whose row stride is a multiple of 8 (the kernels' alignment), copied if not"""
    if t.stride(1) == 1 and t.stride(0) % 8 == 0 and t.data_ptr() % 16 == 0:
        return t
    buf = torch.zeros((t.shape[0], (t.shape[1] + 7) // 8 * 8), dtype=t.dtype, device=t.device)
    buf[:, :t.shape[1]] = t
    return buf[:, :t.shape[1]]


class TcGemm(torch.autograd.Function):
    """gemm() (EPI_NONE) as an autograd op.  Each operand is an fp16 activation (gradient fp16) or the fp16 packed
    copy of an fp32 parameter passed with it (a_param / w_param: the gradient, fp32, goes to the parameter in its own
    layout — Linear (out, in); Conv2d OIHW as a view of the [O][kh][kw][I] result).  The bias (fp32 row or per-batch
    [batch, N]) gets its fp32 gradient, the residual dD.  Positional arguments in tc_gemm()'s order."""

    @staticmethod
    def forward(ctx, a, a_param, w, w_param, bias, residual, a2, bias_batch_stride, rows_per_batch, conv, conv_stride,
                splits, m):
        n = w.shape[0]
        mm = _gemm_m(a, conv, conv_stride, m)
        out = torch.empty((mm, (n + 7) // 8 * 8), dtype=torch.float16, device=a.device)[:, :n]
        gemm(a, w, out=out, bias=bias, bias_batch_stride=bias_batch_stride, rows_per_batch=rows_per_batch,
             residual=residual, a2=a2, conv=conv, conv_stride=conv_stride, splits=splits, m=m)
        ctx.save_for_backward(a, a_param, w, w_param, a2)
        ctx.kw = dict(conv=conv, conv_stride=conv_stride, bias_batch_stride=bias_batch_stride,
                      rows_per_batch=rows_per_batch, m=m)
        ctx.bias_shape = None if bias is None else bias.shape
        ctx.has_residual = residual is not None
        return out

    @staticmethod
    def backward(ctx, dout):
        a, a_param, w, w_param, a2 = ctx.saved_tensors
        dd = _rows8(dout)
        grads = _wanted(ctx, a=(0, 1, 6), b=(2, 3), bias=(4,))
        da, da2, dw, dbias = gemm_backward(
            a, w, dd, a2=a2, grads=grads, da_dtype=torch.float32 if a_param is not None else torch.float16,
            db_dtype=torch.float32 if w_param is not None else torch.float16, **ctx.kw)
        g_a, g_ap = _route_grad(da, a, a_param)
        g_w, g_wp = _route_grad(dw, w, w_param)
        g_bias = dbias.view(ctx.bias_shape) if dbias is not None else None
        g_res = dout if ctx.has_residual else None
        return g_a, g_ap, g_w, g_wp, g_bias, g_res, da2, None, None, None, None, None, None


def tc_gemm(a, w, *, a_param=None, w_param=None, bias=None, bias_batch_stride=0, rows_per_batch=0, residual=None,
            a2=None, conv=None, conv_stride=1, splits=0, m=None, epilogue=EPI_NONE, ln_u=None):
    """Differentiable gemm() (TcGemm).  GEGLU and the folded LayerNorm have no backward kernel and are refused here,
    before anything runs.  Training composes the unfused pieces instead: tc_gemm with proj.weight / proj.bias then
    geglu(), and layer_norm() then tc_gemm (norm2 -> attn2.to_q) — the fold never materialises the normalised rows
    that the weight gradient needs."""
    if epilogue != EPI_NONE:
        raise RuntimeError("magicdance_b200.tc_gemm: the GEGLU epilogue has no backward kernel")
    if ln_u is not None:
        raise RuntimeError("magicdance_b200.tc_gemm: the folded LayerNorm (ln_u) has no backward kernel")
    return TcGemm.apply(a, a_param, w, w_param, bias, residual, a2, bias_batch_stride, rows_per_batch, conv,
                        conv_stride, splits, m)


def _attn_desc(q, k0, vt0, n0, *, heads, d, batch, nq, out, kv0_batches, ldv0_batch, k1, vt1, n1, kv1_batches,
               ldv1_batch, bank_batches, scale):
    for t, nm in ((q, "q"), (k0, "k0"), (vt0, "vt0"), (out, "out")):
        _chk(t, torch.float16, nm)
    a = _lib.AttnDesc()
    a.q, a.ldq = q.data_ptr(), q.stride(0)
    a.k0, a.ldk0, a.vt0, a.ldvt0 = k0.data_ptr(), k0.stride(0), vt0.data_ptr(), vt0.stride(0)
    a.n0 = n0
    a.kv0_batches = batch if kv0_batches is None else kv0_batches
    a.ldv0_batch = n0 if ldv0_batch is None else ldv0_batch
    if n1 > 0:
        _chk(k1, torch.float16, "k1")
        _chk(vt1, torch.float16, "vt1")
        a.k1, a.ldk1, a.vt1, a.ldvt1 = k1.data_ptr(), k1.stride(0), vt1.data_ptr(), vt1.stride(0)
        a.n1, a.kv1_batches = n1, kv1_batches
        a.ldv1_batch = n1 if ldv1_batch is None else ldv1_batch
        a.bank_batches = bank_batches
    a.out, a.ldo = out.data_ptr(), out.stride(0)
    a.batch, a.heads, a.d, a.nq = batch, heads, d, nq
    a.scale = float(d) ** -0.5 if scale is None else scale
    return a


def attention(q, k0, vt0, n0, *, heads, d, batch, nq, out=None, kv0_batches=None, ldv0_batch=None,
              k1=None, vt1=None, n1=0, kv1_batches=1, ldv1_batch=None, bank_batches=0, scale=None, lse=None):
    """softmax([q k0^T | q k1^T] * scale) [v0 ; v1]; k*: [rows, heads*d] (row stride free), vt*: [heads*d, cols].
    lse: optional fp32 [batch, heads, nq] that receives the row log-sum-exp of the scaled scores (natural log), for
    attention_backward; `out` is bit-equal with and without it."""
    lib = _lib.load()
    _chk(q, torch.float16, "q")
    if out is None:
        out = torch.empty((batch * nq, heads * d), dtype=torch.float16, device=q.device)
    a = _attn_desc(q, k0, vt0, n0, heads=heads, d=d, batch=batch, nq=nq, out=out, kv0_batches=kv0_batches,
                   ldv0_batch=ldv0_batch, k1=k1, vt1=vt1, n1=n1, kv1_batches=kv1_batches, ldv1_batch=ldv1_batch,
                   bank_batches=bank_batches, scale=scale)
    if lse is None:
        _lib.check(lib.mdb_attention_f16(C.byref(a), _stream()), "attention_f16")
    else:
        _chk(lse, torch.float32, "lse")
        assert lse.is_contiguous() and lse.numel() == batch * heads * nq
        _lib.check(lib.mdb_attention_lse_f16(C.byref(a), lse.data_ptr(), _stream()), "attention_lse_f16")
    return out


def attention_backward(q, k0, vt0, n0, out, dout, lse, *, heads, d, batch, nq, kv0_batches=None, ldv0_batch=None,
                       k1=None, vt1=None, n1=0, kv1_batches=1, ldv1_batch=None, bank_batches=0, scale=None,
                       out_dq=None, out_dk0=None, out_dvt0=None, out_dk1=None, out_dvt1=None):
    """Gradients of attention() with respect to q, k0, vt0, k1, vt1 from dout (the gradient of `out`), given the
    forward's `out` and `lse`.  Returns (dq, dk0, dvt0, dk1, dvt1) shaped like q, k0, vt0, k1, vt1 (dk1 / dvt1 are
    None without a bank).  Each goes to its out_* tensor when given (fp16, 2-D, unit column stride, row stride a
    multiple of 8); the kernels do not write the padding columns of dvt* nor the bank rows / columns of batch elements
    >= bank_batches, which keep their contents there, and are zero in the new tensors made otherwise.
    Deterministic (csrc/attention_bwd.cu).  Shared sources (kv*_batches == 1 with batch > 1) are not supported."""
    dests = []  # the kernels leave padding columns and unused bank rows unwritten: zeros in the new tensors
    for nm, t, like, zero in (("out_dq", out_dq, q, False), ("out_dk0", out_dk0, k0, False),
                              ("out_dvt0", out_dvt0, vt0, True), ("out_dk1", out_dk1, k1 if n1 > 0 else None, True),
                              ("out_dvt1", out_dvt1, vt1 if n1 > 0 else None, True)):
        if like is None and t is not None:
            raise RuntimeError(f"magicdance_b200: {nm} given without the operand it is the gradient of")
        dests.append(None if like is None else
                     _dest(t, like.shape, torch.float16, q.device, nm, rows8=True, zero=zero))
    dq, dk0, dvt0, dk1, dvt1 = dests
    lib = _lib.load()
    for t, nm in ((q, "q"), (dout, "dout")):
        _chk(t, torch.float16, nm)
    _chk(lse, torch.float32, "lse")
    assert lse.is_contiguous() and lse.numel() == batch * heads * nq
    assert dout.dim() == 2 and dout.stride(1) == 1
    a = _lib.AttnBwdDesc()
    a.fwd = _attn_desc(q, k0, vt0, n0, heads=heads, d=d, batch=batch, nq=nq, out=out, kv0_batches=kv0_batches,
                       ldv0_batch=ldv0_batch, k1=k1, vt1=vt1, n1=n1, kv1_batches=kv1_batches, ldv1_batch=ldv1_batch,
                       bank_batches=bank_batches, scale=scale)
    a.dout, a.lddout, a.lse = dout.data_ptr(), dout.stride(0), lse.data_ptr()
    a.dq, a.lddq = dq.data_ptr(), dq.stride(0)
    a.dk0, a.lddk0, a.dvt0, a.lddvt0 = dk0.data_ptr(), dk0.stride(0), dvt0.data_ptr(), dvt0.stride(0)
    if n1 > 0:
        a.dk1, a.lddk1, a.dvt1, a.lddvt1 = dk1.data_ptr(), dk1.stride(0), dvt1.data_ptr(), dvt1.stride(0)
    ws = _workspace("attn_bwd", int(lib.mdb_attention_bwd_ws_floats(batch, heads, nq)), torch.float32, q.device)
    a.ws = ws.data_ptr()
    _lib.check(lib.mdb_attention_bwd_f16(C.byref(a), _stream()), "attention_bwd_f16")
    return dq, dk0, dvt0, dk1, dvt1


class TwoSourceAttention(torch.autograd.Function):
    """attention() as an autograd op: the forward stores the log-sum-exp, the backward runs attention_backward.
    Positional arguments in the order of attention()'s parameters; two_source_attention() takes them as keywords."""

    @staticmethod
    def forward(ctx, q, k0, vt0, n0, heads, d, batch, nq, kv0_batches=None, ldv0_batch=None, k1=None, vt1=None, n1=0,
                kv1_batches=1, ldv1_batch=None, bank_batches=0, scale=None):
        kw = dict(heads=heads, d=d, batch=batch, nq=nq, kv0_batches=kv0_batches, ldv0_batch=ldv0_batch, k1=k1, vt1=vt1,
                  n1=n1, kv1_batches=kv1_batches, ldv1_batch=ldv1_batch, bank_batches=bank_batches, scale=scale)
        lse = torch.empty((batch, heads, nq), dtype=torch.float32, device=q.device)
        out = attention(q, k0, vt0, n0, lse=lse, **kw)
        ctx.save_for_backward(q, k0, vt0, k1, vt1, out, lse)
        ctx.n0, ctx.kw = n0, {k: v for k, v in kw.items() if k not in ("k1", "vt1")}
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k0, vt0, k1, vt1, out, lse = ctx.saved_tensors
        dq, dk0, dvt0, dk1, dvt1 = attention_backward(q, k0, vt0, ctx.n0, out, dout.contiguous(), lse, k1=k1, vt1=vt1,
                                                      **ctx.kw)
        return (dq, dk0, dvt0) + (None,) * 7 + (dk1, dvt1) + (None,) * 5


def two_source_attention(q, k0, vt0, n0, *, heads, d, batch, nq, kv0_batches=None, ldv0_batch=None, k1=None, vt1=None,
                         n1=0, kv1_batches=1, ldv1_batch=None, bank_batches=0, scale=None):
    """Differentiable attention(): gradients flow to q, k0, vt0, k1 and vt1 (TwoSourceAttention)."""
    return TwoSourceAttention.apply(q, k0, vt0, n0, heads, d, batch, nq, kv0_batches, ldv0_batch, k1, vt1, n1,
                                    kv1_batches, ldv1_batch, bank_batches, scale)


GN_AUTO, GN_TWO_KERNELS, GN_CLUSTER = 0, 1, 2  # mdb_groupnorm_f16 `mode`
GN_DEFAULT_MODE = GN_AUTO


def groupnorm(x1, gamma, beta, *, batch, hw, eps, silu, x2=None, out=None, mode=None):
    """GroupNorm(32) [+SiLU] over [x1 | x2] channels; deterministic, pivot-shifted statistics (csrc/norm.cu)."""
    lib = _lib.load()
    _chk(x1, torch.float16, "x1")
    mode = GN_DEFAULT_MODE if mode is None else mode
    c1 = x1.shape[-1]
    c2 = 0 if x2 is None else x2.shape[-1]
    assert x1.is_contiguous() and (x2 is None or x2.is_contiguous())
    if out is None:
        out = torch.empty((batch * hw, c1 + c2), dtype=torch.float16, device=x1.device)
    # workspace of the two-kernel path (tickets must be zero at first use: _workspace(zero=True)); the single-launch
    # cluster path ignores it
    need = int(lib.mdb_groupnorm_ws_floats(c1 + c2, batch, hw))
    ws = _workspace("gn", need, torch.float32, x1.device, zero=True)
    _lib.check(lib.mdb_groupnorm_f16(x1.data_ptr(), c1, _ptr(x2), c2, gamma.data_ptr(), beta.data_ptr(), out.data_ptr(),
                                     ws.data_ptr(), batch, hw, eps, int(silu), int(mode), _stream()), "groupnorm_f16")
    return out


def layernorm(x, gamma, beta, eps=1e-5, out=None):
    lib = _lib.load()
    _chk(x, torch.float16, "x")
    assert x.is_contiguous()
    rows, c = x.shape
    if out is None:
        out = torch.empty_like(x)
    _lib.check(lib.mdb_layernorm_f16(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), out.data_ptr(), rows, c, eps,
                                     _stream()), "layernorm_f16")
    return out


def groupnorm_backward(x1, gamma, beta, dy, *, batch, hw, eps, silu, x2=None, grads=("x", "gamma", "beta"),
                       dx_dtype=torch.float16, out_dx1=None, out_dx2=None, out_dgamma=None, out_dbeta=None,
                       accumulate=()):
    """Gradients of y = groupnorm(x1, gamma, beta, batch=, hw=, eps=, silu=, x2=) from dy = dL/dy (fp16
    [batch*hw, c1+c2]), csrc/norm_bwd.cu; the statistics are recomputed.  `grads` names the gradients to compute among
    "x" (dx1, and dx2 with x2), "gamma" and "beta".  Each goes to its out_* tensor when given (its dtype is then the
    gradient's dtype) or to a new one of dx_dtype (dgamma / dbeta: fp32); names in `accumulate` ("x", "x2", "gamma",
    "beta") add into the out_* tensor instead of overwriting it.  Returns (dx1, dx2, dgamma, dbeta), None for a
    gradient not requested.  Deterministic.  Groups narrower than 10 channels (the VAE's) are rejected."""
    lib = _lib.load()
    _chk(x1, torch.float16, "x1")
    _chk(dy, torch.float16, "dy")
    _chk(gamma, torch.float32, "gamma")
    _chk(beta, torch.float32, "beta")
    c1 = x1.shape[-1]
    c2 = 0
    if x2 is not None:
        _chk(x2, torch.float16, "x2")
        c2 = x2.shape[-1]
        assert x2.is_contiguous()
    assert x1.is_contiguous() and dy.is_contiguous() and tuple(dy.shape) == (batch * hw, c1 + c2), dy.shape
    dev = x1.device
    d = _lib.GroupNormBwdDesc()
    d.x1, d.x2, d.c1, d.c2 = x1.data_ptr(), _ptr(x2), c1, c2
    d.gamma, d.beta, d.dy = gamma.data_ptr(), beta.data_ptr(), dy.data_ptr()
    d.batch, d.hw, d.eps, d.silu = batch, hw, eps, int(silu)
    acc = set(accumulate)
    dx1 = dx2 = dgamma = dbeta = None
    if "x" in grads:
        dx1 = _dest(out_dx1, (batch * hw, c1), dx_dtype, dev, "out_dx1", any_float=True, contiguous=True)
        d.dx1, d.dx1_dtype, d.dx1_accumulate = dx1.data_ptr(), _DTYPES[dx1.dtype], "x" in acc
        if x2 is not None:
            dx2 = _dest(out_dx2, (batch * hw, c2), dx_dtype, dev, "out_dx2", any_float=True, contiguous=True)
            d.dx2, d.dx2_dtype, d.dx2_accumulate = dx2.data_ptr(), _DTYPES[dx2.dtype], "x2" in acc
    if "gamma" in grads:
        dgamma = _dest(out_dgamma, (c1 + c2,), torch.float32, dev, "out_dgamma", contiguous=True, numel=True)
        d.dgamma, d.dgamma_accumulate = dgamma.data_ptr(), "gamma" in acc
    if "beta" in grads:
        dbeta = _dest(out_dbeta, (c1 + c2,), torch.float32, dev, "out_dbeta", contiguous=True, numel=True)
        d.dbeta, d.dbeta_accumulate = dbeta.data_ptr(), "beta" in acc
    # the statistics kernel's tickets must be zero at first use (_workspace(zero=True)); the kernels leave them so
    d.ws = _bwd_ws(d, lib.mdb_groupnorm_bwd_ws_floats, "gn_bwd", dev, "groupnorm_bwd_f16", zero=True)
    _lib.check(lib.mdb_groupnorm_bwd_f16(C.byref(d), _stream()), "groupnorm_bwd_f16")
    return dx1, dx2, dgamma, dbeta


def layernorm_backward(x, gamma, dy, *, eps=1e-5, grads=("x", "gamma", "beta"), dx_dtype=torch.float16, out_dx=None,
                       out_dgamma=None, out_dbeta=None, accumulate=()):
    """Gradients of y = layernorm(x, gamma, beta, eps) from dy (fp16 [rows, c]), csrc/norm_bwd.cu; mean and rstd are
    recomputed by the forward's code.  grads / out_* / accumulate as in groupnorm_backward ("x", "gamma", "beta").
    Returns (dx, dgamma, dbeta).  Deterministic."""
    lib = _lib.load()
    _chk(x, torch.float16, "x")
    _chk(dy, torch.float16, "dy")
    _chk(gamma, torch.float32, "gamma")
    assert x.is_contiguous() and dy.is_contiguous() and dy.shape == x.shape, (x.shape, dy.shape)
    rows, c = x.shape
    dev = x.device
    d = _lib.LayerNormBwdDesc()
    d.x, d.gamma, d.dy, d.rows, d.c, d.eps = x.data_ptr(), gamma.data_ptr(), dy.data_ptr(), rows, c, eps
    acc = set(accumulate)
    dx = dgamma = dbeta = None
    if "x" in grads:
        dx = _dest(out_dx, (rows, c), dx_dtype, dev, "out_dx", any_float=True, contiguous=True)
        d.dx, d.dx_dtype, d.dx_accumulate = dx.data_ptr(), _DTYPES[dx.dtype], "x" in acc
    if "gamma" in grads:
        dgamma = _dest(out_dgamma, (c,), torch.float32, dev, "out_dgamma", contiguous=True, numel=True)
        d.dgamma, d.dgamma_accumulate = dgamma.data_ptr(), "gamma" in acc
    if "beta" in grads:
        dbeta = _dest(out_dbeta, (c,), torch.float32, dev, "out_dbeta", contiguous=True, numel=True)
        d.dbeta, d.dbeta_accumulate = dbeta.data_ptr(), "beta" in acc
    d.ws = _bwd_ws(d, lib.mdb_layernorm_bwd_ws_floats, "ln_bwd", dev, "layernorm_bwd_f16")
    _lib.check(lib.mdb_layernorm_bwd_f16(C.byref(d), _stream()), "layernorm_bwd_f16")
    return dx, dgamma, dbeta


def _geglu_forward(h):
    lib = _lib.load()
    _chk(h, torch.float16, "h")
    assert h.dim() == 2 and h.stride(1) == 1 and h.shape[1] % 2 == 0
    m, n = h.shape[0], h.shape[1] // 2
    out = torch.empty((m, n), dtype=torch.float16, device=h.device)
    _lib.check(lib.mdb_geglu_f16(h.data_ptr(), h.stride(0), out.data_ptr(), out.stride(0), m, n, _stream()), "geglu_f16")
    return out


def geglu_backward(h, dout):
    """Gradient of out = geglu(h) from dout (fp16 [M, N], row stride a multiple of 8): dh [M, 2N] =
    [dout * gelu(g) | dout * v * gelu'(g)] in the projection's own row order, ready to be gemm_backward's dd."""
    lib = _lib.load()
    _chk(h, torch.float16, "h")
    _chk(dout, torch.float16, "dout")
    assert h.dim() == 2 and h.stride(1) == 1 and dout.dim() == 2 and dout.stride(1) == 1
    m, n = dout.shape
    assert tuple(h.shape) == (m, 2 * n), (h.shape, dout.shape)
    dh = torch.empty((m, 2 * n), dtype=torch.float16, device=h.device)
    _lib.check(lib.mdb_geglu_bwd_f16(h.data_ptr(), h.stride(0), dout.data_ptr(), dout.stride(0), dh.data_ptr(),
                                     dh.stride(0), m, n, _stream()), "geglu_bwd_f16")
    return dh


class GroupNorm(torch.autograd.Function):
    """groupnorm() as an autograd op: fp16 gradients to x1 and x2, fp32 ones to gamma and beta (the nn.Parameters
    themselves, no layout change).  Positional arguments in group_norm()'s order."""

    @staticmethod
    def forward(ctx, x1, gamma, beta, x2, batch, hw, eps, silu):
        ctx.save_for_backward(x1, gamma, beta, x2)
        ctx.kw = dict(batch=batch, hw=hw, eps=eps, silu=silu)
        return groupnorm(x1, gamma, beta, x2=x2, **ctx.kw)

    @staticmethod
    def backward(ctx, dy):
        x1, gamma, beta, x2 = ctx.saved_tensors
        grads = _wanted(ctx, x=(0, 3), gamma=(1,), beta=(2,))
        dx1, dx2, dgamma, dbeta = groupnorm_backward(x1, gamma, beta, dy.contiguous(), x2=x2, grads=grads, **ctx.kw)
        return dx1, dgamma, dbeta, dx2, None, None, None, None


def group_norm(x1, gamma, beta, *, batch, hw, eps, silu, x2=None):
    """Differentiable groupnorm() (GroupNorm): x1 [batch*hw, c1] (and x2 [batch*hw, c2]) fp16, gamma / beta fp32."""
    return GroupNorm.apply(x1, gamma, beta, x2, batch, hw, eps, silu)


class LayerNorm(torch.autograd.Function):
    """layernorm() as an autograd op: an fp16 gradient to x, fp32 ones to gamma and beta."""

    @staticmethod
    def forward(ctx, x, gamma, beta, eps):
        ctx.save_for_backward(x, gamma)
        ctx.eps = eps
        return layernorm(x, gamma, beta, eps)

    @staticmethod
    def backward(ctx, dy):
        x, gamma = ctx.saved_tensors
        grads = _wanted(ctx, x=(0,), gamma=(1,), beta=(2,))
        dx, dgamma, dbeta = layernorm_backward(x, gamma, dy.contiguous(), eps=ctx.eps, grads=grads)
        return dx, dgamma, dbeta, None


def layer_norm(x, gamma, beta, *, eps=1e-5):
    """Differentiable layernorm() (LayerNorm): x fp16 [rows, c], gamma / beta fp32."""
    return LayerNorm.apply(x, gamma, beta, eps)


class Geglu(torch.autograd.Function):
    """The GEGLU activation as an autograd op: out = v * gelu_erf(g) of h = [v | g] (fp16 [M, 2N], the output of a
    plain tc_gemm with proj.weight / proj.bias as they are), gradient dh in the same order."""

    @staticmethod
    def forward(ctx, h):
        ctx.save_for_backward(h)
        return _geglu_forward(h)

    @staticmethod
    def backward(ctx, dout):
        (h,) = ctx.saved_tensors
        return geglu_backward(h, _rows8(dout))


def geglu(h):
    """GEGLU forward (attention.py:53-56) on h = proj(x) in the parameter's row order: fp16 [M, 2N] -> [M, N]
    (csrc/norm_bwd.cu); differentiable (Geglu)."""
    return Geglu.apply(h)


def conv3x3_direct(x, wt, bias, *, batch, h, w, cin, cout, stride=1, silu=False, residual=None, out=None):
    lib = _lib.load()
    _chk(x, torch.float16, "x")
    ho, wo = (h + 2 - 3) // stride + 1, (w + 2 - 3) // stride + 1
    if out is None:
        out = torch.empty((batch * ho * wo, cout), dtype=torch.float16, device=x.device)
    _lib.check(lib.mdb_conv3x3_direct_f16(x.data_ptr(), wt.data_ptr(), _ptr(bias), _ptr(residual), out.data_ptr(), batch,
                                          h, w, cin, cout, stride, int(silu), _stream()), "conv3x3_direct_f16")
    return out


def im2col3x3(x, *, batch, h, w, c, stride, pad="same"):
    """pad='same': one halo pixel on every side (the UNet's convolutions); pad='br': one padding row / column
    at the bottom / right only (the VAE encoder's Downsample, model.py:82-84)"""
    lib = _lib.load()
    _chk(x, torch.float16, "x")
    if pad == "br":
        ho, wo = (h + 1 - 3) // stride + 1, (w + 1 - 3) // stride + 1
        col = torch.empty((batch * ho * wo, 9 * c), dtype=torch.float16, device=x.device)
        _lib.check(lib.mdb_im2col3x3_br_f16(x.data_ptr(), col.data_ptr(), batch, h, w, c, stride, _stream()),
                   "im2col3x3_br_f16")
        return col
    assert pad == "same"
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    col = torch.empty((batch * ho * wo, 9 * c), dtype=torch.float16, device=x.device)
    _lib.check(lib.mdb_im2col3x3_f16(x.data_ptr(), col.data_ptr(), batch, h, w, c, stride, _stream()), "im2col3x3_f16")
    return col


def upsample2x(x, *, batch, h, w, c):
    lib = _lib.load()
    _chk(x, torch.float16, "x")
    y = torch.empty((batch * 4 * h * w, c), dtype=torch.float16, device=x.device)
    _lib.check(lib.mdb_upsample2x_f16(x.data_ptr(), y.data_ptr(), batch, h, w, c, _stream()), "upsample2x_f16")
    return y


def add(a, b, *, batch, b_batches=None, out=None):
    """out = a + b (out may alias a)."""
    lib = _lib.load()
    _chk(a, torch.float16, "a")
    _chk(b, torch.float16, "b")
    assert a.is_contiguous() and b.is_contiguous()
    if out is None:
        out = torch.empty_like(a)
    n_per = a.numel() // batch
    bb = batch if b_batches is None else b_batches
    assert b.numel() == n_per * bb
    _lib.check(lib.mdb_add_f16(a.data_ptr(), b.data_ptr(), out.data_ptr(), n_per, batch, bb, _stream()), "add_f16")
    return out


def timestep_embedding(t, dim, rows=None):
    """rows > len(t): row b uses t[b % len(t)] (one timestep for the whole batch, or the cond | uncond pair)"""
    lib = _lib.load()
    _chk(t, torch.int64, "t")
    assert t.dim() == 1 and t.is_contiguous()
    rows = t.shape[0] if rows is None else rows
    assert rows % t.shape[0] == 0
    out = torch.empty((rows, dim), dtype=torch.float32, device=t.device)
    _lib.check(lib.mdb_timestep_embedding_f32(t.data_ptr(), t.shape[0], out.data_ptr(), rows, dim, _stream()),
               "timestep_embedding_f32")
    return out


def skinny_linear(x, w, bias, *, silu_in=False, silu_out=False):
    lib = _lib.load()
    _chk(x, torch.float32, "x")
    _chk(w, torch.float16, "w")
    rows, k = x.shape
    n = w.shape[0]
    assert w.shape[1] == k and x.is_contiguous() and w.is_contiguous()
    out = torch.empty((rows, n), dtype=torch.float32, device=x.device)
    # the kernel keeps at most 16 activation rows in registers per weight row; taller inputs (more than eight
    # frames per batch, or more than 16 timesteps per bank-build chunk) go through it 16 rows at a time
    for r0 in range(0, rows, SKINNY_MAX_ROWS):
        r = min(SKINNY_MAX_ROWS, rows - r0)
        _lib.check(lib.mdb_skinny_linear_f32(x[r0:].data_ptr(), w.data_ptr(), _ptr(bias), out[r0:].data_ptr(), r, n, k,
                                             int(silu_in), int(silu_out), _stream()), "skinny_linear_f32")
    return out


def softmax_rows(x, scale=1.0):
    """in place: x[r, :] <- softmax(scale * x[r, :]) (fp16 storage, fp32 arithmetic)"""
    lib = _lib.load()
    _chk(x, torch.float16, "x")
    assert x.dim() == 2 and x.stride(1) == 1
    _lib.check(lib.mdb_softmax_rows_f16(x.data_ptr(), x.stride(0), x.shape[0], x.shape[1], float(scale), _stream()),
               "softmax_rows_f16")
    return x


def nchw_f32_to_nhwc_f16(x, out=None, copies=1):
    """copies > 1: the result holds the batch `copies` times over ([copies*B*H*W, C])"""
    lib = _lib.load()
    _chk(x, torch.float32, "x")
    x = x.contiguous()
    b, c, h, w = x.shape
    y = torch.empty((copies * b * h * w, c), dtype=torch.float16, device=x.device) if out is None else out
    _lib.check(lib.mdb_nchw_f32_to_nhwc_f16(x.data_ptr(), y.data_ptr(), b, c, h, w, copies, _stream()),
               "nchw_f32_to_nhwc_f16")
    return y


def nhwc_f16_to_nchw_f32(x, *, batch, c, h, w, out=None):
    lib = _lib.load()
    _chk(x, torch.float16, "x")
    if out is None:
        out = torch.empty((batch, c, h, w), dtype=torch.float32, device=x.device)
    _lib.check(lib.mdb_nhwc_f16_to_nchw_f32(x.data_ptr(), out.data_ptr(), batch, c, h, w, _stream()),
               "nhwc_f16_to_nchw_f32")
    return out


def cfg_ddim_update(x, eps_c, eps_u, coef, noise=None, x_prev=None, pred_x0=None, update_x=False):
    """coef: device fp32[6] = {scale, sqrt(a_t), sqrt(a_prev), sqrt(1-a_prev-sigma^2), sigma, sqrt(1-a_t)};
    update_x: x is overwritten with x_prev as well (the chain advances in place)"""
    lib = _lib.load()
    for t, nm in ((x, "x"), (eps_c, "eps_c"), (eps_u, "eps_u"), (coef, "coef")):
        _chk(t, torch.float32, nm)
    if x_prev is None:
        x_prev = torch.empty_like(x)
    if pred_x0 is None:
        pred_x0 = torch.empty_like(x)
    _lib.check(lib.mdb_cfg_ddim_update_f32(x.data_ptr(), eps_c.data_ptr(), eps_u.data_ptr(), _ptr(noise),
                                           x_prev.data_ptr(), pred_x0.data_ptr(), x.numel(), coef.data_ptr(),
                                           int(update_x), _stream()),
               "cfg_ddim_update_f32")
    return x_prev, pred_x0



# ---------------------------------------------------------------------------------------------------------------------
# Backward of the direct 3x3 conv, the skinny timestep Linear and the nearest x2 upsample (csrc/conv_bwd.cu), and the
# autograd ops over them and over the layout converts.
# ---------------------------------------------------------------------------------------------------------------------
def flip_conv_weight(wt, *, cin, cout):
    """[cout][3][3][cin] -> [cin][2-kh][2-kw][cout] fp16: the weight of the stride-1 dx conv (weight-sized relayout)"""
    return wt.reshape(cout, 3, 3, cin).flip(1, 2).permute(3, 1, 2, 0).contiguous().reshape(cin, 9 * cout)


def conv3x3_direct_backward(x, wt, dy, *, batch, h, w, cin, cout, stride=1, bias=None, silu=False, wt_t=None,
                            grads=("x", "w", "bias"), out_dx=None, out_dw=None, out_dbias=None, accumulate=()):
    """Gradients of y = conv3x3_direct(x, wt, bias, batch=, h=, w=, cin=, cout=, stride=, silu=[, residual=]) from
    dy = dL/dy (fp16 [B*ho*wo, cout]), csrc/conv_bwd.cu; with SiLU the pre-activation is recomputed by the forward
    kernel.  `grads` names the gradients to compute among "x" (fp16 [B*h*w, cin], overwritten), "w" (fp32
    [cout, cin, 3, 3], the Conv2d parameter's OIHW layout) and "bias" (fp32 [cout]); each goes to its out_* tensor
    when given, and names in `accumulate` ("w", "bias") add into it.  wt_t: flip_conv_weight(wt), made here when
    None and needed (stride-1 dx).  The residual's gradient is dy.  Returns (dx, dw, dbias).  Deterministic."""
    lib = _lib.load()
    _chk(x, torch.float16, "x")
    _chk(wt, torch.float16, "wt")
    _chk(dy, torch.float16, "dy")
    assert x.is_contiguous() and wt.is_contiguous() and dy.is_contiguous()
    acc = set(accumulate)
    if "x" in acc:
        raise RuntimeError("magicdance_b200.conv3x3_direct_backward: dx is always overwritten (no accumulation)")
    dev = x.device
    d = _lib.Conv3x3BwdDesc()
    d.x, d.wt, d.dy = x.data_ptr(), wt.data_ptr(), dy.data_ptr()
    if bias is not None:
        _chk(bias, torch.float32, "bias")
        d.bias = bias.data_ptr()
    d.batch, d.h, d.w, d.cin, d.cout, d.stride, d.silu = batch, h, w, cin, cout, stride, int(silu)
    dx = dw = dbias = None
    if "x" in grads:
        if stride == 1:
            wt_t = flip_conv_weight(wt, cin=cin, cout=cout) if wt_t is None else wt_t
            _chk(wt_t, torch.float16, "wt_t")
            assert wt_t.is_contiguous() and wt_t.numel() == wt.numel()
            d.wt_t = wt_t.data_ptr()
        dx = _dest(out_dx, (batch * h * w, cin), torch.float16, dev, "out_dx", contiguous=True)
        d.dx = dx.data_ptr()
    if "w" in grads:
        dw = _dest(out_dw, (cout, cin, 3, 3), torch.float32, dev, "out_dw", contiguous=True, numel=True)
        d.dw, d.dw_accumulate = dw.data_ptr(), "w" in acc
    if "bias" in grads:
        dbias = _dest(out_dbias, (cout,), torch.float32, dev, "out_dbias", contiguous=True, numel=True)
        d.dbias, d.dbias_accumulate = dbias.data_ptr(), "bias" in acc
    d.ws = _bwd_ws(d, lib.mdb_conv3x3_direct_bwd_ws_floats, "conv_bwd", dev, "conv3x3_direct_bwd_f16")
    _lib.check(lib.mdb_conv3x3_direct_bwd_f16(C.byref(d), _stream()), "conv3x3_direct_bwd_f16")
    return dx, dw, dbias


class DirectConv3x3(torch.autograd.Function):
    """conv3x3_direct() as an autograd op: an fp16 gradient to x, fp32 ones to the OIHW parameter w_param (passed with
    its fp16 packed copy wt) and to the bias, dy to the residual.  Only the gradients autograd asks for are computed.
    Positional arguments in direct_conv3x3()'s order."""

    @staticmethod
    def forward(ctx, x, wt, w_param, bias, residual, batch, h, w, cin, cout, stride, silu):
        ctx.kw = dict(batch=batch, h=h, w=w, cin=cin, cout=cout, stride=stride, silu=silu)
        ctx.save_for_backward(x, wt, w_param, bias)
        ctx.has_residual = residual is not None
        return conv3x3_direct(x, wt, bias, residual=residual, **ctx.kw)

    @staticmethod
    def backward(ctx, dy):
        x, wt, w_param, bias = ctx.saved_tensors
        grads = _wanted(ctx, x=(0,), w=(1, 2), bias=(3,))
        dy = dy.contiguous()
        dx = dw = dbias = None
        if grads:
            dx, dw, dbias = conv3x3_direct_backward(x, wt, dy, bias=bias, grads=grads, **ctx.kw)
        g_wt = g_wp = None
        if dw is not None:  # the kernel's dW is OIHW, the parameter's layout
            if w_param is not None:
                g_wp = dw.view(w_param.shape)
            else:
                g_wt = pack_conv_weight(dw).view(wt.shape)
        return dx, g_wt, g_wp, dbias, dy if ctx.has_residual else None, *(None,) * 7


def direct_conv3x3(x, wt, *, batch, h, w, cin, cout, stride=1, silu=False, w_param=None, bias=None, residual=None):
    """Differentiable conv3x3_direct() (DirectConv3x3): x NHWC fp16 [B*h*w, cin], wt fp16 [cout][3][3][cin] (packed
    from the fp32 OIHW w_param, which receives the weight gradient), bias fp32 [cout], residual fp16 like the output."""
    return DirectConv3x3.apply(x, wt, w_param, bias, residual, batch, h, w, cin, cout, stride, silu)


def skinny_linear_backward(x, w, dy, *, silu_in=False, grads=("x", "w", "bias"), out_dx=None, out_dw=None,
                           out_dbias=None, accumulate=()):
    """Gradients of out = skinny_linear(x, w, bias, silu_in=) (silu_out off) from dy (fp32 [rows, n]),
    csrc/conv_bwd.cu: dx fp32 [rows, k] (times silu'(x) with silu_in), dw fp32 [n, k], dbias fp32 [n].  grads / out_* /
    accumulate ("x", "w", "bias") as in gemm_backward.  Inputs taller than SKINNY_MAX_ROWS go through in row chunks, as
    in the forward; dw and dbias of later chunks add onto earlier ones, so the row order of the sums is fixed.
    Returns (dx, dw, dbias).  Deterministic."""
    lib = _lib.load()
    _chk(x, torch.float32, "x")
    _chk(w, torch.float16, "w")
    _chk(dy, torch.float32, "dy")
    rows, k = x.shape
    n = w.shape[0]
    assert w.shape[1] == k and tuple(dy.shape) == (rows, n), (x.shape, w.shape, dy.shape)
    assert x.is_contiguous() and w.is_contiguous() and dy.is_contiguous()
    dev = x.device
    acc = set(accumulate)
    dx = dw = dbias = None
    if "x" in grads:
        dx = _dest(out_dx, (rows, k), torch.float32, dev, "out_dx", contiguous=True)
    if "w" in grads:
        dw = _dest(out_dw, (n, k), torch.float32, dev, "out_dw", contiguous=True)
    if "bias" in grads:
        dbias = _dest(out_dbias, (n,), torch.float32, dev, "out_dbias", contiguous=True, numel=True)
    for r0 in range(0, rows, SKINNY_MAX_ROWS):
        d = _lib.SkinnyBwdDesc()
        d.x, d.w, d.dy = x[r0:].data_ptr(), w.data_ptr(), dy[r0:].data_ptr()
        d.rows, d.n, d.k, d.silu_in = min(SKINNY_MAX_ROWS, rows - r0), n, k, int(silu_in)
        if dx is not None:
            d.dx, d.dx_accumulate = dx[r0:].data_ptr(), "x" in acc
        if dw is not None:
            d.dw, d.dw_accumulate = dw.data_ptr(), r0 > 0 or "w" in acc
        if dbias is not None:
            d.dbias, d.dbias_accumulate = dbias.data_ptr(), r0 > 0 or "bias" in acc
        d.ws = _bwd_ws(d, lib.mdb_skinny_linear_bwd_ws_floats, "skinny_bwd", dev, "skinny_linear_bwd_f32")
        _lib.check(lib.mdb_skinny_linear_bwd_f32(C.byref(d), _stream()), "skinny_linear_bwd_f32")
    return dx, dw, dbias


class SkinnyLinear(torch.autograd.Function):
    """skinny_linear() (silu_out off) as an autograd op: fp32 gradients to x, to the fp32 parameter w_param (passed with
    its fp16 copy w, layout (out, in)) and to the bias.  Positional arguments in skinny_linear_ad()'s order."""

    @staticmethod
    def forward(ctx, x, w, w_param, bias, silu_in):
        ctx.save_for_backward(x, w, w_param)
        ctx.silu_in = silu_in
        return skinny_linear(x, w, bias, silu_in=silu_in)

    @staticmethod
    def backward(ctx, dout):
        x, w, w_param = ctx.saved_tensors
        grads = _wanted(ctx, x=(0,), w=(1, 2), bias=(3,))
        dx = dw = dbias = None
        if grads:
            dx, dw, dbias = skinny_linear_backward(x, w, dout.contiguous(), silu_in=ctx.silu_in, grads=grads)
        g_w, g_wp = _route_grad(dw, w, w_param)
        return dx, g_w, g_wp, dbias, None


def skinny_linear_ad(x, w, bias=None, *, w_param=None, silu_in=False):
    """Differentiable skinny_linear() (SkinnyLinear): x fp32 [rows, k], w fp16 [n, k] (the copy of the fp32 w_param),
    bias fp32 [n].  Training runs time_embed.0 plain and time_embed.2 with silu_in, bit-identical to the fused
    silu_out forward."""
    return SkinnyLinear.apply(x, w, w_param, bias, silu_in)


def upsample2x_backward(dy, *, batch, h, w, c, dx_dtype=torch.float16, out_dx=None, accumulate=False):
    """Gradient of y = upsample2x(x, batch=, h=, w=, c=) from dy (fp16 [B*2h*2w, c]): dx [B*h*w, c] = the 2x2 block
    sums, fp16 or fp32 (out_dx's dtype when given); accumulate adds into out_dx."""
    lib = _lib.load()
    _chk(dy, torch.float16, "dy")
    assert dy.is_contiguous() and tuple(dy.shape) == (batch * 4 * h * w, c), dy.shape
    dx = _dest(out_dx, (batch * h * w, c), dx_dtype, dy.device, "out_dx", any_float=True, contiguous=True)
    _lib.check(lib.mdb_upsample2x_bwd_f16(dy.data_ptr(), dx.data_ptr(), _DTYPES[dx.dtype], int(accumulate), batch, h,
                                          w, c, _stream()), "upsample2x_bwd_f16")
    return dx


class Upsample2x(torch.autograd.Function):
    """upsample2x() (nearest x2, NHWC fp16) as an autograd op: the gradient is the 2x2 block sum."""

    @staticmethod
    def forward(ctx, x, batch, h, w, c):
        ctx.kw = dict(batch=batch, h=h, w=w, c=c)
        return upsample2x(x, **ctx.kw)

    @staticmethod
    def backward(ctx, dy):
        return upsample2x_backward(dy.contiguous(), **ctx.kw), None, None, None, None


def upsample_2x(x, *, batch, h, w, c):
    """Differentiable upsample2x() (Upsample2x): x fp16 [B*h*w, c] -> [B*2h*2w, c]."""
    return Upsample2x.apply(x, batch, h, w, c)


class NchwToNhwc(torch.autograd.Function):
    """nchw_f32_to_nhwc_f16() (one copy) as an autograd op; the gradient is the opposite convert."""

    @staticmethod
    def forward(ctx, x):
        ctx.shape = tuple(x.shape)
        return nchw_f32_to_nhwc_f16(x)

    @staticmethod
    def backward(ctx, dy):
        b, c, h, w = ctx.shape
        return nhwc_f16_to_nchw_f32(dy.contiguous(), batch=b, c=c, h=h, w=w)


def nchw_to_nhwc(x):
    """Differentiable nchw_f32_to_nhwc_f16() (NchwToNhwc): NCHW fp32 -> NHWC fp16 [B*H*W, C]."""
    return NchwToNhwc.apply(x)


class NhwcToNchw(torch.autograd.Function):
    """nhwc_f16_to_nchw_f32() as an autograd op; the gradient is the opposite convert."""

    @staticmethod
    def forward(ctx, x, batch, c, h, w):
        return nhwc_f16_to_nchw_f32(x, batch=batch, c=c, h=h, w=w)

    @staticmethod
    def backward(ctx, dy):
        return nchw_f32_to_nhwc_f16(dy.contiguous()), None, None, None, None


def nhwc_to_nchw(x, *, batch, c, h, w):
    """Differentiable nhwc_f16_to_nchw_f32() (NhwcToNchw): NHWC fp16 [B*H*W, C] -> NCHW fp32."""
    return NhwcToNchw.apply(x, batch, c, h, w)


class Add(torch.autograd.Function):
    """add() of two same-shaped fp16 tensors as an autograd op (the pose residuals onto the UNet's skips); both
    gradients are dy."""

    @staticmethod
    def forward(ctx, a, b, batch):
        return add(a, b, batch=batch)

    @staticmethod
    def backward(ctx, dy):
        return dy, dy, None


def add_ad(a, b, *, batch):
    """Differentiable add() (Add): a + b, fp16, contiguous, same shape (one b per batch element)."""
    return Add.apply(a, b, batch)
