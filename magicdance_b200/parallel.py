"""Multi-GPU partition of the denoising path (SURVEY §8e): frames are independent 50-step chains
from the same x_T (test_tiktok.py:225,232-268), so they are sharded across ranks with no
collective inside a step.  The ONE exchange is the appearance bank: with wonoise it depends on
(reference latent, timestep) only, so the timesteps are dealt round-robin over the ranks, each
rank runs the appearance 'write' pass + K/V projection for its share, and a single NCCL
all-gather at sequence start gives every rank every timestep's bank K/V.

One process per GPU (torchrun); torch.distributed is plumbing (NCCL on GPUs, gloo in CPU tests).
"""
from __future__ import annotations

from typing import Callable, Dict, List, Sequence, Tuple

import torch
import torch.distributed as dist


def shard_frames(n_frames: int, world: int, rank: int) -> range:
    """Contiguous block of frames of this rank (64 frames / 8 ranks -> 8 each; remainders to low ranks)."""
    base, rem = divmod(n_frames, world)
    start = rank * base + min(rank, rem)
    return range(start, start + base + (1 if rank < rem else 0))


def shard_timesteps(indices: Sequence[int], world: int, rank: int) -> List[int]:
    """Round-robin deal of DDIM indices (50 steps / 8 ranks -> 7,7,6,6,6,6,6,6)."""
    return [ix for j, ix in enumerate(indices) if j % world == rank]


def owner_slot(indices: Sequence[int], world: int) -> Dict[int, Tuple[int, int]]:
    """ddim index -> (owning rank, slot in that rank's local buffer)."""
    out = {}
    for j, ix in enumerate(indices):
        out[ix] = (j % world, j // world)
    return out


class BankLayout:
    """Flat fp16 layout of one timestep's bank K/V: per attention layer K [rows, C] then V^T [C, ldv], ldv = rows
    rounded up to a multiple of 8 (the attention kernels' V^T column alignment; the padding columns are never read).
    Every block starts 16-byte aligned (C is a multiple of 8).  Where every layer's rows are a multiple of 8 (every
    level of a 512x512 image) V^T is [C, rows] and the layout is unpadded."""

    def __init__(self, layer_shapes: Sequence[Tuple[int, int]]):
        self.layer_shapes = list(layer_shapes)  # (rows = ref_batches * N_l, C_l)
        self.ldv = [(rows + 7) // 8 * 8 for rows, _ in self.layer_shapes]
        self.offsets = []
        off = 0
        for (rows, c), ldv in zip(self.layer_shapes, self.ldv):
            self.offsets.append(off)
            off += rows * c + c * ldv
        self.numel = (off + 127) // 128 * 128

    def views(self, flat: torch.Tensor, tokens_per_batch: Sequence[int], batches: int):
        """flat [numel] -> list of (K, V^T, N_l, batches) tuples aliasing the buffer, V^T [C, ldv] (project_bank's
        tuples: each sample's V^T column block is V^T.shape[1] // batches wide)."""
        res = []
        for (rows, c), ldv, off, n in zip(self.layer_shapes, self.ldv, self.offsets, tokens_per_batch):
            # per-sample blocks of ldv // batches columns: one sample, or tokens already a multiple of 8
            assert rows == n * batches and ldv == batches * ((n + 7) // 8 * 8), (rows, n, batches)
            k = flat[off:off + rows * c].view(rows, c)
            vt = flat[off + rows * c:off + rows * c + c * ldv].view(c, ldv)
            res.append((k, vt, n, batches))
        return res


def bank_storage(slots: int, layout: BankLayout, device, world: int = 1):
    """(local [slots, numel], gathered [slots, world, numel] or None) fp16 buffers for build_and_gather_bank: row s of
    `gathered` is the contiguous destination of the all-gather of every rank's slot s"""
    local = torch.zeros((slots, layout.numel), dtype=torch.float16, device=device)
    gathered = torch.empty((slots, world, layout.numel), dtype=torch.float16, device=device) if world > 1 else None
    return local, gathered



def bank_chunk_size(n_timesteps: int, world: int, max_chunk: int = 25) -> int:
    """Timesteps per appearance-pass launch: a rank's share of the sequence's timesteps (ceil(n/world)) is
    split into equal chunks of at most `max_chunk` (50 -> 25+25, 25 -> 25, 13 -> 13, 7 -> 7).  Equal, because
    the captured bank-build graph has a fixed batch and a short last chunk would be padded to full size."""
    per_rank = max(1, (n_timesteps + world - 1) // world)
    n_chunks = (per_rank + max_chunk - 1) // max_chunk
    return (per_rank + n_chunks - 1) // n_chunks

class GatheredBank:
    """ddim index -> flat fp16 bank buffer, plus the handles of the exchange that fills it.

    The timesteps are dealt round-robin in CONSUMPTION order, so slot s of every rank together holds the timesteps
    the steps s*world ... (s+1)*world-1 need: the exchange is issued as one all-gather PER SLOT ROW, in that order,
    and a step only waits for its own row (`wait(index)`); the remaining rows travel over NVLink while the first
    steps already run.  `dict`-like for the callers that only need index -> buffer."""

    def __init__(self, table, works=None, slot_of=None):
        # works: slot row -> c10d work handle of its all-gather
        self.table, self.works, self.slot_of = table, works or {}, slot_of or {}
        self._waited = set()

    def __getitem__(self, ix):
        return self.table[ix]

    def __iter__(self):
        return iter(self.table)

    def __len__(self):
        return len(self.table)

    def items(self):
        return self.table.items()

    def wait(self, ix=None):
        """make the CURRENT stream wait for the gather that delivers ddim index ix (all of them if None)"""
        slots = list(self.works) if ix is None else [self.slot_of.get(ix)]
        for s_ in slots:
            if s_ is not None and s_ in self.works and s_ not in self._waited:
                self.works[s_].wait()
                self._waited.add(s_)


def build_and_gather_bank(indices: Sequence[int], layout: BankLayout,
                          build_fn: Callable[[List[int], torch.Tensor], None], device, world: int = 1, rank: int = 0,
                          group=None, chunk: int = 10, storage=None, timing=None) -> GatheredBank:
    """Each rank calls build_fn(ddim_indices_chunk, slots[len(chunk), numel]) for its share of `indices`
    (build_fn fills the flat fp16 slots in place; chunks of up to `chunk` timesteps are built as ONE
    batched appearance pass), then the slots are exchanged: one all_gather_into_tensor per slot row, issued
    asynchronously in consumption order (see GatheredBank).  Returns ddim index -> flat buffer (views into the
    gathered storage); call .wait(index) before reading one.  timing: optional dict that receives CUDA events
    ('build0', 'build1') recorded around this rank's build."""
    mine = shard_timesteps(indices, world, rank)
    slots = (len(indices) + world - 1) // world
    if storage is not None:  # (local, gathered) preallocated by bank_storage(): keeps cudaMalloc out of timed regions
        if storage[0].shape[0] != slots:
            raise ValueError(f"bank storage holds {storage[0].shape[0]} slots per rank, this exchange needs {slots}: "
                             "allocate it with bank_storage(slots, ...) for the sequence length at hand")
        local, gathered = storage
    else:
        local, gathered = bank_storage(slots, layout, device, world)
    ev = (lambda: None)
    if timing is not None and torch.device(device).type == "cuda":
        def ev(name=None):
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            return e
        timing["build0"] = ev()
    for s0 in range(0, len(mine), chunk):
        part = mine[s0:s0 + chunk]
        build_fn(part, local[s0:s0 + len(part)])
    if timing is not None and "build0" in timing:
        timing["build1"] = ev()
    if world == 1:
        return GatheredBank({ix: local[s] for s, ix in enumerate(mine)})
    table = owner_slot(indices, world)
    flat_of = {ix: gathered[s, r] for ix, (r, s) in table.items()}
    slot_of = {ix: s for ix, (r, s) in table.items()}
    works = {}
    for s in range(slots):
        works[s] = dist.all_gather_into_tensor(gathered[s].view(-1), local[s], group=group, async_op=True)
    return GatheredBank(flat_of, works, slot_of)
