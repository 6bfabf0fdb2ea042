"""Output poisoning for the kernel numerics cases.

A case that hands a kernel a fresh `torch.empty` cannot see an element the kernel never writes: on CUDA the caching
allocator returns the block the previous case just freed, which may already hold the right answer.  Nor can it see a
write outside the output, nor a read of operand padding that happens to be zero.  These helpers close the three gaps:

- `Guarded`: the output lives inside a NaN-filled buffer with guard rows above and below and guard columns on both
  sides.  After the launch every interior element must be finite (it was written) and every guard element must still
  hold the sentinel's exact bits (nothing was written there).
- `poisoned_alloc` / `check_poisoned`: for ops that allocate their own result, the block the op will get from the
  allocator is filled with the sentinel first.
- `block_rel` / `gated`: rel-L2 per output block, so that an error confined to one tile is not averaged away by
  the rest.
- `poison_workspace`: the op's scratch buffer holds the sentinel, so a read of scratch the kernel has not written
  yet shows as NaN.

CPU-only code: tests/test_kernel_edges_cpu.py checks that the checks catch what they are meant to catch."""
import torch

# NaN bit patterns with a payload that no arithmetic produces (canonical NaNs are 0x7e00 / 0x7fc00000)
SENTINEL = {torch.float16: (torch.int16, 0x7E5A), torch.float32: (torch.int32, 0x7FC5A5A5)}

# Per-block gate: the worst block's rel-L2 may reach BLOCK_FACTOR x the case's tolerance.  Measured on an H100 80GB
# HBM3 (700 W power limit) over the 190 gated cases of tests/kernel_cases.py, the worst block of any case was 0.14 x
# its tolerance (4.3e-4 against 3e-3, folded LayerNorm at M = 1); the global rel-L2 of those cases reaches 0.1 x.
# A factor of 2 leaves that natural spread far below the gate and still fails an error confined to one tile that
# the whole-output rel-L2 averages away.  On the same card, over the 178 gated backward cases (tests/gemm_bwd_cases.py,
# attention_bwd_cases.py, norm_bwd_cases.py), the worst block was 1.17 x its tolerance (attention dq at d = 160 with
# a near one-hot softmax, where dS = P (dP - D) cancels); outside the sharp-softmax cases the worst was 0.64 x
# (attention, one query), and 0.2 x outside attention.
BLOCK_FACTOR = 2.0


def poison_(t):
    """fills t (fp16 / fp32, any view) with the sentinel NaN in place; returns t"""
    idt, bits = SENTINEL[t.dtype]
    t.view(idt).fill_(bits)
    return t


class Guarded:
    """A [rows, cols] output inside a sentinel-filled buffer: `top` / `bottom` guard rows and, unless `contiguous`,
    `left` guard columns and at least `right` on the right (the row pitch is rounded up to 8 elements).  The interior
    `out` keeps 16-byte alignment and a row stride that is a multiple of 8; with `contiguous` it is a dense tensor
    (row stride cols), for kernels that take a bare pointer, and `shape` reshapes it."""

    def __init__(self, rows, cols, dtype=torch.float16, *, contiguous=False, top=8, bottom=128, left=8, right=8,
                 shape=None, keep=None, device="cuda"):
        """keep: optional bool [rows, cols] mask of interior elements the kernel must NOT write (the padding columns
        of a per-sample V^T block, the bank rows of samples without a bank); check() treats them as guard elements"""
        if contiguous:
            left, right, ld = 0, 0, cols
        else:
            assert left % 8 == 0
            ld = left + (cols + 7) // 8 * 8 + right
        assert top % 8 == 0  # top * ld elements of 2 or 4 bytes keep the interior 16-byte aligned
        self.buf = poison_(torch.empty((top + rows + bottom, ld), dtype=dtype, device=device))
        self.guard = torch.ones(self.buf.shape, dtype=torch.bool, device=device)
        self.guard[top:top + rows, left:left + cols] = False
        if keep is not None:
            assert tuple(keep.shape) == (rows, cols)
            self.guard[top:top + rows, left:left + cols] = keep.to(device)
        out = self.buf[top:top + rows, left:left + cols]
        self.out = out if shape is None else out.view(shape)
        assert self.out.data_ptr() % 16 == 0 and (contiguous or ld % 8 == 0)

    def check(self, what="output"):
        """asserts that every interior element outside `keep` was written (is finite) and that no guard or `keep`
        element was"""
        idt, bits = SENTINEL[self.buf.dtype]
        stray = (self.buf.view(idt) != bits) & self.guard
        if bool(stray.any()):
            r, c = (int(i) for i in stray.nonzero()[0])
            raise AssertionError(f"{what}: {int(stray.sum())} guard elements overwritten, the first at buffer row {r} "
                                 f"column {c} (value {float(self.buf[r, c])})")
        check_finite(self.buf[~self.guard], what)


def check_finite(t, what="output"):
    bad = ~torch.isfinite(t)
    if bool(bad.any()):
        raise AssertionError(f"{what}: {int(bad.sum())} of {t.numel()} elements not finite (never written, or NaN / "
                             f"Inf from poisoned padding), the first at flat index {int(bad.reshape(-1).nonzero()[0])}")


def poisoned_alloc(shape, dtype, device="cuda"):
    """Fills the block the caching allocator will hand to the next allocation of this size with the sentinel and
    returns its address.  The allocation and the free leave the free lists as they were, so the op's own
    `torch.empty` of the same byte size on the same stream gets that block back; check_poisoned asserts it did."""
    t = poison_(torch.empty(shape, dtype=dtype, device=device))
    ptr = t.data_ptr()
    del t
    return ptr


def check_poisoned(result, ptr, what="result"):
    """the op's result must occupy the poisoned block (else the test proves nothing) and be fully written"""
    assert result.data_ptr() == ptr, (f"{what}: the allocator did not hand back the poisoned block (got "
                                      f"{result.data_ptr():#x}, poisoned {ptr:#x}); the unwritten-element check "
                                      f"cannot run")
    check_finite(result, what)


def bit_equal(a, b):
    """a and b hold the same bits (torch.equal is False wherever both hold the same NaN, e.g. the sentinel an
    output must keep)"""
    idt = SENTINEL[a.dtype][0]
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(idt), b.view(idt))


def poison_workspace(key, need=0, device="cuda"):
    """Fills the op's scratch buffer `key` (ops._workspace, grown to at least `need` fp32 elements) with the
    sentinel and returns it, for the workspaces documented as needing no initial value ("gemm_bwd", "attn_bwd",
    "ln_bwd"; not "gn_bwd", whose tickets must start at zero).  A kernel that reads an element before writing it
    turns its result into NaN.  The op reuses the buffer as long as its own need is not larger;
    check_workspace_used asserts that it did."""
    from magicdance_b200 import ops
    return poison_(ops._workspace(key, need, torch.float32, _op_device(device)))


def check_workspace_used(key, buf, what="output", device="cuda"):
    from magicdance_b200 import ops
    cur = ops._ws_cache.get((key, _op_device(device), ops.current_lane()))
    assert cur is buf, f"{what}: the op outgrew the poisoned {key!r} workspace; the poisoned run proves nothing"


def _op_device(device):
    """the device as an op's operand reports it (ops._workspace keys on tensor.device, which carries the index)"""
    d = torch.device(device)
    return torch.device(d.type, torch.cuda.current_device()) if d.type == "cuda" and d.index is None else d


def rel(a, b):
    """rel-L2 of a against the reference b, in float64"""
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    return float((a - b).norm() / (b.norm() + 1e-30))


def gated(out, ref, tol, rows=128, cols=32, groups=1):
    """(error, note): the rel-L2 of the whole output, or the worst block's (block_rel) over BLOCK_FACTOR when that is
    larger, so that err <= tol gates both"""
    g, b = rel(out, ref), block_rel(out, ref, rows, cols, groups)
    return max(g, b / BLOCK_FACTOR), f" [rel-L2 {g:.2e}, worst block {b:.2e} = {b / tol:.2f} tol]"


def block_rel(out, ref, rows, cols, groups=1):
    """The worst rel-L2 over blocks of `rows` x `cols` elements.  out / ref: [groups * R, C] (or anything of that
    many elements); the blocks tile each group's [R, C] matrix from its first row, the last block of a ragged edge
    being partial (attention: one group per sample, 64 queries x one head per block)."""
    o = out.double().reshape(groups, -1, ref.shape[-1])
    r = ref.double().reshape(groups, -1, ref.shape[-1])
    g, rr, cc = r.shape
    pr, pc = -rr % rows, -cc % cols
    diff = torch.nn.functional.pad(o - r, (0, pc, 0, pr))
    refp = torch.nn.functional.pad(r, (0, pc, 0, pr))
    shape = (g, (rr + pr) // rows, rows, (cc + pc) // cols, cols)
    num = diff.reshape(shape).pow(2).sum((2, 4))
    den = refp.reshape(shape).pow(2).sum((2, 4))
    return float((num.sqrt() / (den.sqrt() + 1e-30)).max())
