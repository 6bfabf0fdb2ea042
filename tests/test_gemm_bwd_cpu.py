"""CPU-only checks of the GEMM backward's C ABI: descriptor layout, compiled resources, argument rejection before any
launch, no CPU fallback, and a well-formed GPU case list."""
import ctypes as C
import os
import re
import subprocess

import pytest
import torch

from tests.test_attention_bwd_cpu import _kernels

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_gemm_bwd_desc_matches_the_ctypes_struct(tmp_path):
    """mdb_gemm_bwd_desc has exactly the layout magicdance_b200/_lib.py declares (compiled as C99)"""
    from magicdance_b200 import _lib
    inc = os.path.join(REPO, "include")
    cls = _lib.GemmBwdDesc
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "magicdance_b200.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(mdb_gemm_bwd_desc));']
    lines += [f'  printf("{f} %zu\\n", offsetof(mdb_gemm_bwd_desc, {f}));' for f, _ in cls._fields_]
    lines += ['  return 0;', '}']
    src = tmp_path / "abi.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "abi"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", inc, str(src), "-o", str(exe)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["size"]) == C.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(got[f]) == getattr(cls, f).offset, f
    assert _lib.load().mdb_abi_struct_bytes(3) == C.sizeof(cls)


def test_backward_kernels_do_not_spill_and_run_on_wgmma():
    from magicdance_b200 import build
    usage, bodies = _kernels(build.build())
    gemm = sorted(n for n in usage if "gemm_bwd_kernel" in n)
    assert len(gemm) == 2, gemm  # dA (MN-major B) and dB (both operands MN-major)
    for name in gemm:
        assert re.search(r"HGMMA\.\S+ .*tnsp[AB]", bodies[name]), f"{name}: no MN-major (transposed) wgmma operand"
        assert "UTMALDG" in bodies[name], name
    both = [n for n in gemm if "ILi1E" in n]
    assert both and re.search(r"HGMMA\.\S+ .*tnspA.*tnspB|HGMMA\.\S+ .*tnspB.*tnspA", bodies[both[0]]), \
        "dB reads both operands MN-major"
    helpers = [n for n in usage if re.search(r"gemm_bwd_finalize|col2im_gather|colsum_(partial|finalize)", n)]
    assert len(helpers) == 4, helpers
    for name in gemm + helpers:
        assert usage[name] == (0, 0), f"{name}: LOCAL / STACK = {usage[name]}"


def _desc(**over):
    """a plain 256 x 320 x 320 backward descriptor whose pointers are never dereferenced: the argument checks run
    before any CUDA call"""
    from magicdance_b200 import _lib
    g = _lib.GemmBwdDesc()
    f = g.fwd
    f.a, f.lda, f.k1, f.b, f.ldb = 0x10000, 320, 320, 0x20000, 320
    f.m, f.n, f.k = 256, 320, 320
    g.dd, g.lddd = 0x30000, 320
    g.da, g.ldda, g.db, g.lddb, g.db_dtype = 0x40000, 320, 0x50000, 320, 1
    g.ws = 0x60000
    for k, v in over.items():
        setattr(f if k.startswith("fwd_") else g, k.removeprefix("fwd_"), v)
    return g


@pytest.mark.parametrize("over,msg", [
    (dict(fwd_epilogue=1), "GEGLU"),
    (dict(fwd_ln_u=0x70000), "ln_u"),
    (dict(fwd_conv=1, fwd_nb=1, fwd_h=16, fwd_w=16, fwd_c=64, fwd_k=640), "k == 9c"),
    (dict(fwd_conv=1, fwd_nb=1, fwd_h=16, fwd_w=16, fwd_c=64, fwd_k=576, fwd_a2=0x70000), "single source"),
    (dict(fwd_conv=3, fwd_nb=1, fwd_h=16, fwd_w=16, fwd_c=64, fwd_k=576), "conv must be 1 or 2"),
    (dict(fwd_conv=1, fwd_nb=1, fwd_h=16, fwd_w=16, fwd_c=64, fwd_k=576, fwd_m=200), "m != nb"),
    (dict(fwd_k=100), "bad shape"),
    (dict(lddd=100), "lddd"),
    (dict(dd=0x30002), "lddd"),
    (dict(ldda=321), "da must be"),
    (dict(db_dtype=2), "db must be"),
])
def test_backward_rejects_before_any_launch(over, msg):
    """GEGLU, the folded LayerNorm, conv geometry no path takes and misalignment are refused with a message, with or
    without a GPU, and nothing is launched"""
    from magicdance_b200 import _lib
    lib = _lib.load()
    n0 = lib.mdb_launch_count()
    g = _desc(**over)
    assert lib.mdb_gemm_bwd_f16(C.byref(g), None) == -1
    assert msg.replace("%", "") in lib.mdb_last_error().decode().replace("%", "")
    assert lib.mdb_gemm_bwd_ws_floats(C.byref(g)) == -1
    assert lib.mdb_launch_count() == n0


def test_workspace_size():
    """split slabs and the column buffers are sized from the same plan the launch uses"""
    from magicdance_b200 import _lib
    lib = _lib.load()
    g = _desc(splits=4)  # dB over M = 256 rows: 4 chunks, one per split -> fp32 slabs [4][N][K]
    g.fwd.splits = 1
    assert lib.mdb_gemm_bwd_ws_floats(C.byref(g)) == 4 * 320 * 320
    g = _desc(splits=1)
    g.fwd.splits = 1
    assert lib.mdb_gemm_bwd_ws_floats(C.byref(g)) == 0
    # a 12x8 latent (no TMA boxes): dA's fp32 column buffer [M][9c]
    g = _desc(fwd_conv=1, fwd_nb=1, fwd_h=12, fwd_w=8, fwd_c=64, fwd_k=576, fwd_m=96, fwd_n=64, db=None, lddd=64,
              fwd_splits=1)
    assert lib.mdb_gemm_bwd_ws_floats(C.byref(g)) == 96 * 576


def test_backward_has_no_cpu_fallback():
    from magicdance_b200 import ops
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    a = torch.zeros(128, 64).half()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.gemm_backward(a, a, a)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.tc_gemm(a, a)


def test_geglu_and_ln_u_are_refused_by_the_autograd_op():
    from magicdance_b200 import ops
    a = torch.zeros(128, 64).half()
    with pytest.raises(RuntimeError, match="GEGLU"):
        ops.tc_gemm(a, a, epilogue=ops.EPI_GEGLU)
    with pytest.raises(RuntimeError, match="ln_u"):
        ops.tc_gemm(a, a, ln_u=torch.zeros(128))


def test_backward_case_list_is_well_formed():
    """the GPU-side case list binds to its case function (a typo must not cost GPU time)"""
    import inspect
    from tests import gemm_bwd_cases as G
    sig = inspect.signature(G.case_gemm_bwd)
    for kw in G.CASES:
        sig.bind(**kw)
    assert len({G.case_id(kw) for kw in G.CASES}) == len(G.CASES)
