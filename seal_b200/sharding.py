"""Multi-GPU: query sharding with replicated index + weights and ONE gather of result records.

Queries are independent (own beams, SA ranges, hypotheses); the FM-index and BART weights are
read-only, so every rank (one process per GPU) decodes a contiguous block of the batch and the
fixed-size hypothesis records are gathered once to rank 0 — the only collective (SURVEY.md §8e).

The records of a rank live in ONE contiguous byte buffer (`RecordLayout`): the decode kernels write
scores / lengths / tokens / validity / SA ranges straight into it on the device, and that buffer is what
the collective moves — one `dist.gather` (NCCL on the GPUs, device to device over NVLink; gloo on CPU
tensors in the tests), no packing pass, no host bounce.  This module is numpy/torch only.
"""
from typing import Callable, Dict, List, Optional

import numpy as np

# field -> (numpy dtype, trailing shape as a function of T); order = descending alignment
_FIELDS = (("lo", np.uint64, False), ("hi", np.uint64, False), ("scores", np.float32, False),
           ("lens", np.int32, False), ("tokens", np.int32, True), ("valid", np.uint8, False))
HEADER_BYTES = 16          # int64 n_queries actually filled, int64 reserved
ERR_BYTES = 16             # int32[4] error flags of the generate call (include/sealdec.h)


def shard_bounds(n: int, world: int, rank: int):
    """Contiguous block [lo, hi) of rank `rank`; blocks differ by at most one query."""
    base, extra = divmod(n, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


class RecordLayout:
    """Byte layout of the hypothesis records of up to `n_queries` queries (H hypotheses each, T tokens per
    hypothesis): [header | lo | hi | scores | lens | tokens | valid | pad | err].  Every field starts 16-byte
    aligned; `nbytes` is what one rank contributes to the gather."""

    def __init__(self, n_queries: int, hyps: int, max_length: int):
        self.Q, self.H, self.T = int(n_queries), int(hyps), int(max_length)
        off = HEADER_BYTES
        self.offsets = {}
        for name, dt, has_t in _FIELDS:
            shape = (self.Q, self.H, self.T) if has_t else (self.Q, self.H)
            nb = int(np.prod(shape)) * np.dtype(dt).itemsize
            self.offsets[name] = (off, np.dtype(dt), shape, nb)
            off += (nb + 15) // 16 * 16
        self.err_offset = off
        self.nbytes = off + ERR_BYTES
        self.record_bytes = sum(v[3] for v in self.offsets.values())

    def views(self, buf: np.ndarray) -> Dict[str, np.ndarray]:
        """Typed numpy views into a host copy of the buffer (uint8 array of `nbytes`)."""
        out = {}
        for name, (off, dt, shape, nb) in self.offsets.items():
            out[name] = buf[off:off + nb].view(dt).reshape(shape)
        return out

    def n_filled(self, buf: np.ndarray) -> int:
        return int(buf[:8].view(np.int64)[0])

    def errors(self, buf: np.ndarray) -> np.ndarray:
        return buf[self.err_offset:self.err_offset + ERR_BYTES].view(np.int32)


def pack_host_records(rec: Dict[str, np.ndarray], layout: RecordLayout, n_local: int) -> np.ndarray:
    """Host-side filler (CPU tests / tools): dict of per-query arrays -> one layout buffer."""
    buf = np.zeros(layout.nbytes, dtype=np.uint8)
    buf[:8] = np.asarray([n_local], dtype=np.int64).view(np.uint8)
    v = layout.views(buf)
    for name in v:
        if rec.get(name) is not None and n_local:
            v[name][:n_local] = rec[name][:n_local]
    return buf


def gather_buffers(buf, dst: int = 0, group=None):
    """THE collective: every rank's layout buffer (a 1-D uint8 torch tensor, CUDA or CPU) to rank `dst`.
    Returns the list of world_size buffers on `dst`, None elsewhere."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group); rank = dist.get_rank(group)
    out = [torch.empty_like(buf) for _ in range(world)] if rank == dst else None
    dist.gather(buf, out, dst=dst, group=group)
    return out


def merge_gathered(bufs: List, layout: RecordLayout) -> Dict[str, np.ndarray]:
    """Rank-ordered buffers -> full-batch record arrays (host), plus 'errors' = elementwise max of the ranks' flags."""
    merged = {name: [] for name in layout.offsets}
    errs = np.zeros(4, dtype=np.int32)
    for t in bufs:
        raw = t.cpu().numpy() if hasattr(t, "cpu") else np.asarray(t)
        n = layout.n_filled(raw)
        v = layout.views(raw)
        for name in merged:
            merged[name].append(v[name][:n])
        errs = np.maximum(errs, layout.errors(raw))
    out = {k: np.concatenate(v, axis=0) for k, v in merged.items()}
    out["errors"] = errs
    return out


def sharded_generate(fill_fn: Callable, input_ids, attention_mask, hyps: int, max_length: int, group=None,
                     dst: int = 0) -> Optional[Dict[str, np.ndarray]]:
    """Decode this rank's block of the batch and gather the records to rank `dst` with one collective.

    `fill_fn(ids_block, mask_block, layout) -> 1-D uint8 torch tensor of layout.nbytes` holding the block's
    records in `layout` (header filled).  On the GPUs that is `seal_b200.beam_search.DeviceRecords` filled by the
    decode kernels (`fill_device_records`); the CPU tests pass a numpy stand-in.  Every rank's layout is sized
    for the largest block so the collective is a plain gather of equal buffers.
    Returns the full-batch records on `dst`, None elsewhere."""
    import torch.distributed as dist
    world = dist.get_world_size(group); rank = dist.get_rank(group)
    n = len(input_ids)
    lo, hi = shard_bounds(n, world, rank)
    n_max = max(shard_bounds(n, world, r)[1] - shard_bounds(n, world, r)[0] for r in range(world))
    layout = RecordLayout(max(n_max, 1), hyps, max_length)
    buf = fill_fn(input_ids[lo:hi], attention_mask[lo:hi], layout)
    bufs = gather_buffers(buf, dst=dst, group=group)
    if bufs is None:
        return None
    return merge_gathered(bufs, layout)
