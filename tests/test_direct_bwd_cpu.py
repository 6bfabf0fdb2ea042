"""CPU-only checks of the direct-conv / skinny-Linear / upsample backward C ABI: descriptor layouts, compiled resources,
argument rejection before any launch, no CPU fallback, and a well-formed GPU case list."""
import ctypes as C
import os
import subprocess

import pytest
import torch

from tests.test_attention_bwd_cpu import _kernels

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("struct,cls_name,which", [("mdb_conv3x3_bwd_desc", "Conv3x3BwdDesc", 6),
                                                   ("mdb_skinny_linear_bwd_desc", "SkinnyBwdDesc", 7)])
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
    keys = ("conv3x3_dw_kernel", "conv3x3_s2_dx_kernel", "silu_grad_kernel", "skinny_bwd_dx", "skinny_bwd_dw",
            "upsample2x_bwd")
    names = [n for n in usage if any(k in n for k in keys)]
    # dW at stride 1 / 2, stride-2 dx, dz, skinny dx at 2 / 8 / 16 rows + its finalize, skinny dW at 2 / 8 / 16 rows,
    # upsample
    assert len(names) == 12, names
    for name in names:
        assert usage[name] == (0, 0), f"{name}: LOCAL / STACK = {usage[name]}"


def _conv(**over):
    """a 2 x 64 x 64, 16 -> 32 stride-2 SiLU conv backward descriptor whose pointers are never dereferenced: the
    argument checks run before any CUDA call"""
    from magicdance_b200 import _lib
    d = _lib.Conv3x3BwdDesc()
    d.x, d.wt, d.wt_t, d.bias, d.dy = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000
    d.batch, d.h, d.w, d.cin, d.cout, d.stride, d.silu = 2, 64, 64, 16, 32, 2, 1
    d.dx, d.dw, d.dbias, d.ws = 0x60000, 0x70000, 0x80000, 0x90000
    for k, v in over.items():
        setattr(d, k, v)
    return d


def _skinny(**over):
    from magicdance_b200 import _lib
    d = _lib.SkinnyBwdDesc()
    d.x, d.w, d.dy, d.rows, d.n, d.k, d.silu_in = 0x10000, 0x20000, 0x30000, 4, 20160, 1280, 1
    d.dx, d.dw, d.dbias, d.ws = 0x40000, 0x50000, 0x60000, 0x70000
    for k, v in over.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("over,msg", [
    (dict(x=None), "null pointer"),
    (dict(dy=None), "null pointer"),
    (dict(stride=3), "stride must be 1 or 2"),
    (dict(cin=0), "bad shape"),
    (dict(batch=0), "bad shape"),
    (dict(h=-1), "bad shape"),
    (dict(dx=None, dw=None, dbias=None), "no gradient requested"),
    (dict(dy=0x50004), "16B aligned"),
    (dict(dx=0x60002), "dx must be 16B aligned"),
    (dict(stride=1, wt_t=None), "flipped weight"),
    (dict(stride=1, wt_t=0x30008), "flipped weight"),
])
def test_conv_backward_rejects_before_any_launch(over, msg):
    from magicdance_b200 import _lib
    lib = _lib.load()
    n0 = lib.mdb_launch_count()
    d = _conv(**over)
    assert lib.mdb_conv3x3_direct_bwd_f16(C.byref(d), None) == -1
    assert msg in lib.mdb_last_error().decode()
    assert lib.mdb_conv3x3_direct_bwd_ws_floats(C.byref(d)) == -1
    assert lib.mdb_launch_count() == n0


@pytest.mark.parametrize("over,msg", [
    (dict(w=None), "null pointer"),
    (dict(rows=17), "bad shape"),
    (dict(rows=0), "bad shape"),
    (dict(k=1284), "bad shape"),
    (dict(dx=None, dw=None, dbias=None), "no gradient requested"),
    (dict(dw=0x50004), "16B aligned"),
])
def test_skinny_backward_rejects_before_any_launch(over, msg):
    from magicdance_b200 import _lib
    lib = _lib.load()
    n0 = lib.mdb_launch_count()
    d = _skinny(**over)
    assert lib.mdb_skinny_linear_bwd_f32(C.byref(d), None) == -1
    assert msg in lib.mdb_last_error().decode()
    assert lib.mdb_skinny_linear_bwd_ws_floats(C.byref(d)) == -1
    assert lib.mdb_launch_count() == n0


@pytest.mark.parametrize("args,msg", [
    ((None, 0x20000, 0, 0, 2, 8, 8, 640), "null pointer"),
    ((0x10000, 0x20000, 0, 0, 2, 8, 8, 636), "bad shape"),
    ((0x10000, 0x20000, 0, 0, 0, 8, 8, 640), "bad shape"),
    ((0x10008, 0x20000, 0, 0, 2, 8, 8, 640), "16B aligned"),
    ((0x10000, 0x20000, 2, 0, 2, 8, 8, 640), "dx_dtype"),
])
def test_upsample_backward_rejects_before_any_launch(args, msg):
    from magicdance_b200 import _lib
    lib = _lib.load()
    n0 = lib.mdb_launch_count()
    assert lib.mdb_upsample2x_bwd_f16(*args, None) == -1
    assert msg in lib.mdb_last_error().decode()
    assert lib.mdb_launch_count() == n0


def test_workspace_size():
    """conv: the fp16 pre-activation (SiLU only), then dW and dbias slabs for the gradients wanted; skinny: the dX
    slabs only"""
    from magicdance_b200 import _lib
    lib = _lib.load()
    ws = lambda **o: lib.mdb_conv3x3_direct_bwd_ws_floats(C.byref(_conv(**o)))
    z = 2 * 32 * 32 * 32 // 2  # B ho wo cout halves
    assert ws(dw=None, dbias=None) == z
    assert ws(silu=0, dw=None, dbias=None) == 0
    full, no_w = ws(), ws(dw=None)
    assert full > no_w > z and (no_w - z) % 32 == 0 and (full - no_w) % (32 * 9 * 16) == 0
    sk = lambda **o: lib.mdb_skinny_linear_bwd_ws_floats(C.byref(_skinny(**o)))
    assert sk(dx=None) == 0
    assert sk() > 0 and sk() % (4 * 1280) == 0


def test_backward_has_no_cpu_fallback():
    from magicdance_b200 import ops
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    x = torch.zeros(64, 16).half()
    wt = torch.zeros(32, 144).half()
    dy = torch.zeros(16, 32).half()
    xf, wf = torch.zeros(4, 1280), torch.zeros(320, 1280).half()
    for call in (lambda: ops.conv3x3_direct_backward(x, wt, dy, batch=1, h=8, w=8, cin=16, cout=32, stride=2),
                 lambda: ops.direct_conv3x3(x, wt, batch=1, h=8, w=8, cin=16, cout=32),
                 lambda: ops.skinny_linear_backward(xf, wf, torch.zeros(4, 320)),
                 lambda: ops.skinny_linear_ad(xf, wf),
                 lambda: ops.upsample2x_backward(torch.zeros(256, 16).half(), batch=1, h=8, w=8, c=16),
                 lambda: ops.upsample_2x(x, batch=1, h=8, w=8, c=16),
                 lambda: ops.nchw_to_nhwc(torch.zeros(1, 4, 8, 8)),
                 lambda: ops.nhwc_to_nchw(x, batch=1, c=16, h=8, w=8)):
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            call()


def test_backward_case_list_is_well_formed():
    """the GPU-side case list binds to its case functions (a typo must not cost GPU time)"""
    import inspect
    from tests import direct_bwd_cases as N
    for fn, kw in N.CASES:
        inspect.signature(fn).bind(**kw)
    assert len({N.case_id(c) for c in N.CASES}) == len(N.CASES)
