"""CPU-only checks of the attention backward's C ABI: descriptor layout, compiled resources, argument rejection."""
import ctypes as C
import os
import re
import subprocess

import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_bwd_desc_matches_the_ctypes_struct(tmp_path):
    """mdb_attn_bwd_desc has exactly the layout magicdance_b200/_lib.py declares (compiled as C99)"""
    from magicdance_b200 import _lib
    inc = os.path.join(REPO, "include")
    cls = _lib.AttnBwdDesc
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "magicdance_b200.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(mdb_attn_bwd_desc));']
    lines += [f'  printf("{f} %zu\\n", offsetof(mdb_attn_bwd_desc, {f}));' for f, _ in cls._fields_]
    lines += ['  return 0;', '}']
    src = tmp_path / "abi.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "abi"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", inc, str(src), "-o", str(exe)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["size"]) == C.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(got[f]) == getattr(cls, f).offset, f
    assert _lib.load().mdb_abi_struct_bytes(2) == C.sizeof(cls)


def _kernels(path):
    """{mangled name: (LOCAL, STACK)} of every kernel in the library, and {mangled name: SASS text}"""
    res = subprocess.run(["cuobjdump", "--dump-resource-usage", path], capture_output=True, text=True, check=True).stdout
    usage = {}
    lines = res.splitlines()
    for i, line in enumerate(lines):
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            use = dict(re.findall(r"(STACK|LOCAL):(\d+)", lines[i + 1]))
            usage[m.group(1)] = (int(use["LOCAL"]), int(use["STACK"]))
    sass = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    bodies = dict(re.findall(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", sass, re.S))
    return usage, bodies


def test_backward_kernels_do_not_spill_and_run_on_wgmma():
    from magicdance_b200 import build
    usage, bodies = _kernels(build.build())
    bwd = sorted(n for n in usage if "attn_bwd" in n)
    # dQ for d = 40 / 80 / 160; dK+dV for d = 40 / 80; dV and dK passes for d = 160
    assert len(bwd) == 7, bwd
    for name in bwd:
        assert usage[name] == (0, 0), f"{name}: LOCAL / STACK = {usage[name]}"
        assert "HGMMA" in bodies[name], name
        assert re.search(r"HGMMA\.\S+ .*tnsp[AB]", bodies[name]), f"{name}: no MN-major (transposed) wgmma operand"
    lse = [n for n in usage if "attn_wg_kernel" in n]
    assert len(lse) == 8 and all(usage[n] == (0, 0) for n in lse), lse


def _fake_bwd_desc(batch, kv0_batches, kv1_batches, n1):
    """a descriptor whose pointers are never dereferenced: the argument checks run before any CUDA call"""
    from magicdance_b200 import _lib
    a = _lib.AttnBwdDesc()
    f = a.fwd
    f.q, f.k0, f.vt0, f.out = 0x10000, 0x20000, 0x30000, 0x40000
    f.ldq = f.ldk0 = f.ldo = f.ldk1 = 320
    f.ldvt0, f.ldvt1 = batch * 64, 64 * max(kv1_batches, 1)
    f.n0, f.kv0_batches, f.ldv0_batch = 64, kv0_batches, 64
    f.k1, f.vt1, f.n1, f.kv1_batches, f.ldv1_batch = 0x50000, 0x60000, n1, kv1_batches, 64
    f.batch, f.heads, f.d, f.nq, f.bank_batches, f.scale = batch, 8, 40, 64, batch, 40 ** -0.5
    a.dout, a.lddout, a.lse, a.ws = 0x70000, 320, 0x80000, 0x90000
    a.dq, a.lddq, a.dk0, a.lddk0, a.dvt0, a.lddvt0 = 0xa0000, 320, 0xb0000, 320, 0xc0000, batch * 64
    a.dk1, a.lddk1, a.dvt1, a.lddvt1 = 0xd0000, 320, 0xe0000, 64
    return a


@pytest.mark.parametrize("which", [0, 1])
def test_backward_rejects_shared_sources_before_any_launch(which):
    """kv*_batches == 1 with batch > 1 would need a reduction across batch elements: refused with a message, with or
    without a GPU"""
    from magicdance_b200 import _lib
    lib = _lib.load()
    n0 = lib.mdb_launch_count()
    a = _fake_bwd_desc(2, 1 if which == 0 else 2, 1 if which == 1 else 2, 64)
    assert lib.mdb_attention_bwd_f16(C.byref(a), None) == -1
    assert f"shared source {which}" in lib.mdb_last_error().decode()
    assert lib.mdb_launch_count() == n0
    assert lib.mdb_attention_bwd_ws_floats(2, 8, 64) == 2 * 8 * 64


def test_backward_has_no_cpu_fallback():
    from magicdance_b200 import ops
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    q = torch.zeros(64, 320).half()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.attention_backward(q, q, q.t().contiguous(), 64, q, q, torch.zeros(1, 8, 64), heads=8, d=40, batch=1,
                               nq=64)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.two_source_attention(q, q, q.t().contiguous(), 64, heads=8, d=40, batch=1, nq=64)


def test_backward_case_list_is_well_formed():
    """the GPU-side case list binds to its case function (a typo must not cost GPU time)"""
    import inspect
    from tests import attention_bwd_cases as A
    sig = inspect.signature(A.case_attention_bwd)
    for args in A.CASES:
        sig.bind(**args) if isinstance(args, dict) else sig.bind(*args)
    assert len({A.case_id(a) for a in A.CASES}) == len(A.CASES)


def _cpu_operands():
    q = torch.zeros(64, 320).half()
    return q, dict(heads=8, d=40, batch=1, nq=64)


@pytest.mark.parametrize("name, bad, match", [
    ("out_dq", lambda q: torch.zeros(64, 320), "2-D float16"),                        # fp32
    ("out_dk0", lambda q: torch.zeros(320, 64).half().t(), "unit column stride"),     # transposed
    ("out_dk0", lambda q: torch.zeros(64, 324).half()[:, :320], "multiple of 8"),    # row stride 324
    ("out_dvt0", lambda q: torch.zeros(320, 72).half(), "shape \\(320, 64\\)"),    # wrong width
    ("out_dq", lambda q: torch.zeros(1, 64, 320).half(), "2-D"),
    ("out_dk1", lambda q: torch.zeros(64, 320).half(), "without the operand"),       # no bank (n1 = 0)
])
def test_backward_output_buffers_are_validated_before_any_launch(name, bad, match):
    """out_dq / out_dk0 / out_dvt0 / out_dk1 / out_dvt1 of ops.attention_backward: fp16, 2-D, unit column stride,
    the operand's shape, a row stride that is a multiple of 8; refused with a message before the library is asked
    to do anything, with or without a GPU"""
    from magicdance_b200 import ops
    q, kw = _cpu_operands()
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match=match):
        ops.attention_backward(q, q, q.t().contiguous(), 64, q, q, torch.zeros(1, 8, 64), **kw, **{name: bad(q)})
    assert ops.launch_count() == n0


def test_backward_takes_valid_output_buffers_up_to_the_device_check():
    """well-formed out_* buffers (a row stride wider than the row) pass the validation; on a machine without a GPU
    the call then stops at the CUDA-tensor check"""
    from magicdance_b200 import ops
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    q, kw = _cpu_operands()
    outs = dict(out_dq=torch.zeros(64, 336).half()[:, :320], out_dk0=torch.zeros(64, 320).half(),
                out_dvt0=torch.zeros(320, 64).half())
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.attention_backward(q, q, q.t().contiguous(), 64, q, q, torch.zeros(1, 8, 64), **kw, **outs)
