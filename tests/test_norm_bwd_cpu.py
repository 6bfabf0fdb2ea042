"""CPU-only checks of the GroupNorm / LayerNorm / GEGLU backward C ABI: descriptor layouts, compiled resources, argument
rejection before any launch, no CPU fallback, and a well-formed GPU case list."""
import ctypes as C
import os
import subprocess

import pytest
import torch

from tests.test_attention_bwd_cpu import _kernels

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("struct,cls_name,which", [("mdb_groupnorm_bwd_desc", "GroupNormBwdDesc", 4),
                                                   ("mdb_layernorm_bwd_desc", "LayerNormBwdDesc", 5)])
def test_desc_matches_the_ctypes_struct(tmp_path, struct, cls_name, which):
    """each descriptor has exactly the layout magicdance_b200/_lib.py declares (compiled as C99)"""
    from magicdance_b200 import _lib
    inc = os.path.join(REPO, "include")
    cls = getattr(_lib, cls_name)
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "magicdance_b200.h"', 'int main(void) {',
             f'  printf("size %zu\\n", sizeof({struct}));']
    lines += [f'  printf("{f} %zu\\n", offsetof({struct}, {f}));' for f, _ in cls._fields_]
    lines += ['  return 0;', '}']
    src = tmp_path / "abi.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "abi"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", inc, str(src), "-o", str(exe)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["size"]) == C.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(got[f]) == getattr(cls, f).offset, f
    assert _lib.load().mdb_abi_struct_bytes(which) == C.sizeof(cls)


def test_backward_kernels_do_not_spill():
    from magicdance_b200 import build
    usage, _ = _kernels(build.build())
    names = [n for n in usage if any(k in n for k in ("gn_bwd_reduce", "gn_bwd_apply", "layernorm_bwd", "geglu"))]
    assert len(names) == 7, names  # GroupNorm reduce + apply, LayerNorm at 320 / 640 / 1280, GEGLU fwd + bwd
    for name in names:
        assert usage[name] == (0, 0), f"{name}: LOCAL / STACK = {usage[name]}"


def _gn(**over):
    """a 4 x 1024 x (640 + 320) GroupNorm backward descriptor whose pointers are never dereferenced: the argument
    checks run before any CUDA call"""
    from magicdance_b200 import _lib
    d = _lib.GroupNormBwdDesc()
    d.x1, d.x2, d.c1, d.c2 = 0x10000, 0x20000, 640, 320
    d.gamma, d.beta, d.dy = 0x30000, 0x40000, 0x50000
    d.batch, d.hw, d.eps, d.silu = 4, 1024, 1e-5, 1
    d.dx1, d.dx2, d.dgamma, d.dbeta, d.ws = 0x60000, 0x70000, 0x80000, 0x90000, 0xa0000
    for k, v in over.items():
        setattr(d, k, v)
    return d


def _ln(**over):
    from magicdance_b200 import _lib
    d = _lib.LayerNormBwdDesc()
    d.x, d.gamma, d.dy, d.rows, d.c, d.eps = 0x10000, 0x20000, 0x30000, 4096, 640, 1e-5
    d.dx, d.dgamma, d.dbeta, d.ws = 0x40000, 0x50000, 0x60000, 0x70000
    for k, v in over.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("over,msg", [
    (dict(c1=128, x2=None, c2=0), "4-channel groups"),       # the first-stage VAE's 128-channel level
    (dict(c1=256, x2=None, c2=0), "8-channel groups"),
    (dict(c1=2560, c2=320), "unsupported width 2880"),
    (dict(c1=644, c2=316), "multiples of 8"),
    (dict(c2=0), "x2 and c2"),
    (dict(x1=None), "null pointer"),
    (dict(dy=0x50008), "16B aligned"),
    (dict(dx1=0x60004), "dx1 must be"),
    (dict(dx2_dtype=2), "dx2 must be"),
    (dict(batch=0), "bad shape"),
    (dict(batch=2048), "bad shape"),
])
def test_groupnorm_backward_rejects_before_any_launch(over, msg):
    from magicdance_b200 import _lib
    lib = _lib.load()
    n0 = lib.mdb_launch_count()
    d = _gn(**over)
    assert lib.mdb_groupnorm_bwd_f16(C.byref(d), None) == -1
    assert msg in lib.mdb_last_error().decode()
    assert lib.mdb_groupnorm_bwd_ws_floats(C.byref(d)) == -1
    assert lib.mdb_launch_count() == n0


@pytest.mark.parametrize("over,msg", [
    (dict(c=768), "unsupported width 768"),
    (dict(c=2560), "unsupported width 2560"),
    (dict(x=None), "null pointer"),
    (dict(dy=0x30002), "16B aligned"),
    (dict(dx=0x40008), "dx must be"),
    (dict(dx_dtype=3), "dx must be"),
    (dict(rows=0), "bad shape"),
])
def test_layernorm_backward_rejects_before_any_launch(over, msg):
    from magicdance_b200 import _lib
    lib = _lib.load()
    n0 = lib.mdb_launch_count()
    d = _ln(**over)
    assert lib.mdb_layernorm_bwd_f16(C.byref(d), None) == -1
    assert msg in lib.mdb_last_error().decode()
    assert lib.mdb_layernorm_bwd_ws_floats(C.byref(d)) == -1
    assert lib.mdb_launch_count() == n0


@pytest.mark.parametrize("args,msg", [
    ((0x10000, 2560, 0x20000, 1280, 1024, 1284), "n % 8 == 0"),
    ((0x10008, 2560, 0x20000, 1280, 1024, 1280), "h must be"),
    ((0x10000, 2000, 0x20000, 1280, 1024, 1280), "ldh >= 2n"),
    ((0x10000, 2560, 0x20004, 1280, 1024, 1280), "must be 16B aligned"),
    ((0x10000, 2560, None, 1280, 1024, 1280), "must be 16B aligned"),
])
def test_geglu_rejects_before_any_launch(args, msg):
    """the forward's (h, ldh, out, ldo, m, n) and the backward's (h, ldh, dout, lddout, m, n) with dh = dout's slot
    shifted: misalignment and bad shapes are refused with a message"""
    from magicdance_b200 import _lib
    lib = _lib.load()
    n0 = lib.mdb_launch_count()
    h, ldh, out, ldo, m, n = args
    assert lib.mdb_geglu_f16(h, ldh, out, ldo, m, n, None) == -1
    assert msg in lib.mdb_last_error().decode().replace("%%", "%")
    assert lib.mdb_geglu_bwd_f16(h, ldh, out, ldo, 0x40000, 2 * ldo, m, n, None) == -1
    assert lib.mdb_launch_count() == n0


def test_workspace_size():
    """GroupNorm: the statistics kernel's region, A / B [2][batch][c] and the per-CTA slabs; LayerNorm: slabs only
    when a parameter gradient is wanted"""
    from magicdance_b200 import _lib
    lib = _lib.load()
    d = _gn()
    stats = lib.mdb_groupnorm_ws_floats(960, 4, 1024)
    nblk = (stats - 1024 - 4 * 64) // (4 * 64)
    assert lib.mdb_groupnorm_bwd_ws_floats(C.byref(d)) == stats + 2 * 4 * 960 + 2 * 4 * nblk * 960
    assert lib.mdb_layernorm_bwd_ws_floats(C.byref(_ln(dgamma=None, dbeta=None))) == 0
    assert lib.mdb_layernorm_bwd_ws_floats(C.byref(_ln())) > 0


def test_backward_has_no_cpu_fallback():
    from magicdance_b200 import ops
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    x = torch.zeros(256, 320).half()
    g = torch.ones(320)
    for call in (lambda: ops.groupnorm_backward(x, g, g, x, batch=1, hw=256, eps=1e-5, silu=True),
                 lambda: ops.layernorm_backward(x, g, x),
                 lambda: ops.geglu_backward(x, x[:, :160]),
                 lambda: ops.geglu(x),
                 lambda: ops.group_norm(x, g, g, batch=1, hw=256, eps=1e-5, silu=True),
                 lambda: ops.layer_norm(x, g, g)):
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            call()


def test_backward_case_list_is_well_formed():
    """the GPU-side case list binds to its case functions (a typo must not cost GPU time)"""
    import inspect
    from tests import norm_bwd_cases as N
    for fn, kw in N.CASES:
        inspect.signature(fn).bind(**kw)
    assert len({N.case_id(c) for c in N.CASES}) == len(N.CASES)
