"""CPU checks of the kernel tests' own machinery (tests/kernel_guard.py) and of argument checks that refuse bad
input before any launch."""
import ctypes as C
import inspect

import pytest
import torch

from tests import kernel_guard as KG


def test_block_gate_catches_one_scaled_tile_that_the_global_gate_passes():
    g = torch.Generator().manual_seed(0)
    ref = torch.randn(65536, 320, generator=g)
    out = ref.clone()
    out[4096:4224, 96:128] *= 1.05
    assert KG.rel(out, ref) < 2e-3  # ~7e-4: the whole-output rel-L2 alone would pass
    assert KG.block_rel(out, ref, 128, 32) == pytest.approx(0.05, rel=1e-6)
    err, _ = KG.gated(out, ref, 2e-3)
    assert err > 2e-3


def test_block_rel_tiles_each_group_from_its_first_row():
    """attention blocks: 64 queries of one sample x one head; a ragged nq must not merge two samples' rows"""
    ref = torch.ones(2 * 65, 16)
    out = ref.clone()
    out[65] = 2.0  # first query of sample 1: alone in the second sample's first block with 63 clean rows
    assert KG.block_rel(out, ref, 64, 8, groups=2) == pytest.approx((8 / (64 * 8)) ** 0.5)


def _filled(rows, cols, **kw):
    gb = KG.Guarded(rows, cols, device="cpu", **kw)
    gb.out.copy_(torch.randn(rows, cols).half())
    return gb


@pytest.mark.parametrize("contiguous", [False, True])
def test_guard_catches_a_single_stray_zero(contiguous):
    gb = _filled(129, 77, contiguous=contiguous)
    gb.check()
    assert gb.out.data_ptr() % 16 == 0 and (contiguous or gb.buf.stride(0) % 8 == 0)
    # row 129 of the interior's column 0: the first row past M of a ragged tile
    gb.buf[8 + 129, 0 if contiguous else 8] = 0.0
    with pytest.raises(AssertionError, match="1 guard elements overwritten"):
        gb.check()


def test_guard_sees_writes_by_bits_not_by_value():
    """a kernel that writes a NaN of its own into the guard is caught, although NaN != NaN either way"""
    gb = _filled(16, 40)
    gb.buf[0, 0] = float("nan")
    with pytest.raises(AssertionError, match="guard elements overwritten"):
        gb.check()


def test_guard_catches_an_unwritten_element():
    gb = _filled(128, 64)
    KG.poison_(gb.out[127, 63:])
    with pytest.raises(AssertionError, match="1 of 8192 elements not finite"):
        gb.check()


def test_guard_columns_between_width_and_pitch():
    gb = KG.Guarded(4, 72, torch.float32, right=24, device="cpu")
    assert gb.out.stride(0) == 8 + 72 + 24
    gb.out.fill_(1.0)
    gb.check()
    gb.buf[2, 8 + 72] = 1.0
    with pytest.raises(AssertionError):
        gb.check()


def test_poisoned_allocation_must_come_back():
    t = KG.poison_(torch.empty(4, 8))
    with pytest.raises(AssertionError, match="did not hand back the poisoned block"):
        KG.check_poisoned(torch.zeros(4, 8), t.data_ptr())
    with pytest.raises(AssertionError, match="not finite"):
        KG.check_poisoned(t, t.data_ptr())


def test_edge_case_lists_are_well_formed():
    """the GPU-side case lists bind to their case functions (a typo must not cost GPU time)"""
    from tests import kernel_edge_cases as E
    for fn, args in E.EDGE_CASES:
        inspect.signature(fn).bind(*args)


def test_attention_rejects_unaligned_bank_sample_stride_before_any_launch():
    """the V^T tensor map steps from sample to sample by ldv1_batch columns: TMA needs 16-byte strides"""
    from magicdance_b200 import _lib
    lib = _lib.load()
    a = _lib.AttnDesc()
    a.q, a.k0, a.vt0, a.out, a.k1, a.vt1 = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000, 0x60000
    a.ldq = a.ldk0 = a.ldo = a.ldk1 = 320
    a.ldvt0, a.ldvt1 = 2 * 64, 2 * 72
    a.n0, a.kv0_batches, a.ldv0_batch = 64, 2, 64
    a.n1, a.kv1_batches, a.bank_batches = 65, 2, 2
    a.batch, a.heads, a.d, a.nq, a.scale = 2, 8, 40, 64, 40 ** -0.5
    n0 = lib.mdb_launch_count()
    for ldv1 in (65, 68):
        a.ldv1_batch = ldv1
        assert lib.mdb_attention_f16(C.byref(a), None) == -1
        assert "ldv1_batch must be >= n1 and % 8" in lib.mdb_last_error().decode()
    assert lib.mdb_launch_count() == n0


def _vt_with_keep(n=77, ldv=80, batch=2, rows=40):
    """a dvt-like Guarded [rows, batch*ldv] whose padding columns n..ldv of each sample must not be written"""
    keep = torch.zeros(rows, batch * ldv, dtype=torch.bool)
    for b in range(batch):
        keep[:, b * ldv + n:(b + 1) * ldv] = True
    gb = KG.Guarded(rows, batch * ldv, keep=keep, device="cpu")
    for b in range(batch):
        gb.out[:, b * ldv:b * ldv + n] = torch.randn(rows, n).half()
    return gb


def test_keep_mask_passes_when_only_the_allowed_elements_are_written():
    gb = _vt_with_keep()
    gb.check()
    assert torch.isnan(gb.out[:, 77:80]).all()  # the keep-out columns still hold the sentinel


def test_keep_mask_catches_a_single_write_into_a_keep_out_column():
    gb = _vt_with_keep()
    gb.out[5, 80 + 78] = 0.0  # sample 1's padding column 78
    with pytest.raises(AssertionError, match="1 guard elements overwritten, the first at buffer row 13 column 166"):
        gb.check()


def test_keep_mask_catches_a_single_unwritten_element():
    gb = _vt_with_keep()
    KG.poison_(gb.out[39, 80 + 76:80 + 77])  # sample 1's last key of the last row
    with pytest.raises(AssertionError, match="1 of 6160 elements not finite"):
        gb.check()


def test_keep_mask_covers_whole_rows():
    """the bank rows of samples >= bank_batches (dk1)"""
    keep = torch.zeros(200, 320, dtype=torch.bool)
    keep[100:] = True
    gb = KG.Guarded(200, 320, keep=keep, device="cpu")
    gb.out[:100] = 1.0
    gb.check()
    gb.out[150, 7] = 1.0
    with pytest.raises(AssertionError, match="1 guard elements overwritten"):
        gb.check()


def test_poisoned_workspace_is_the_one_the_op_gets():
    from magicdance_b200 import ops
    key = "kernel_guard_selftest"
    ws = KG.poison_workspace(key, 100, device="cpu")
    assert ws.numel() >= 100 and bool((ws.view(torch.int32) == KG.SENTINEL[torch.float32][1]).all())
    assert ops._workspace(key, 50, torch.float32, torch.device("cpu")) is ws
    KG.check_workspace_used(key, ws, device="cpu")
    ops._workspace(key, 10 * ws.numel(), torch.float32, torch.device("cpu"))  # an op that needs more regrows it
    with pytest.raises(AssertionError, match="outgrew the poisoned"):
        KG.check_workspace_used(key, ws, device="cpu")
    ops._ws_cache.pop((key, torch.device("cpu"), ops.current_lane()))


def test_bit_equal_compares_nan_payloads():
    a = KG.poison_(torch.empty(4, 8).half())
    b = a.clone()
    assert not torch.equal(a, b) and KG.bit_equal(a, b)
    b[0, 0] = float("nan")  # a canonical NaN is not the sentinel
    assert not KG.bit_equal(a, b)
