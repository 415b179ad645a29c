# -*- coding: utf-8 -*-
"""Multi-GPU execution: shard the signal-batch axis, one process per GPU.

The reference has no distributed code (SURVEY section 8e); the path shards
embarrassingly over dim 0 of a 2-D input (`_cwt.py:27-28`: rows are independent
signals).  Each rank recomputes the tiny host parameters identically, transforms
its contiguous slice of the batch and keeps its outputs on its own GPU.  The only
collective is an OPTIONAL final `all_gather` of the outputs (NCCL over NVLink);
it moves orders of magnitude more bytes than the compute touches, so it is off
by default and timed separately in the benchmarks.
"""
import torch
import torch.distributed as dist

__all__ = ['shard_bounds', 'ssq_cwt_sharded', 'gather_batch']


def shard_bounds(B, rank, world):
    """Contiguous [lo, hi) slice of a batch of B for `rank` (first B % world ranks
    get one extra signal); empty slices are allowed when B < world."""
    if world < 1 or not (0 <= rank < world):
        raise ValueError("bad rank/world: %s/%s" % (rank, world))
    base, extra = divmod(int(B), world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def gather_batch(local, B, group=None):
    """all_gather of per-rank output shards (dim 0 ragged) -> full [B, ...] tensor
    on every rank."""
    world = dist.get_world_size(group)
    sizes = [shard_bounds(B, r, world) for r in range(world)]
    mx = max(hi - lo for lo, hi in sizes)
    pad_shape = (mx,) + tuple(local.shape[1:])
    buf = local.new_zeros(pad_shape)
    buf[:local.shape[0]] = local
    parts = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(parts, buf, group=group)
    return torch.cat([p[:hi - lo] for p, (lo, hi) in zip(parts, sizes)], dim=0)


def ssq_cwt_sharded(x, *args, gather=False, group=None, _compute=None, get_Wx=True, **kw):
    """`ssq_cwt` on this rank's slice of the batch `x` ([B, N], identical on every
    rank).  Returns `(Tx, Wx, ssq_freqs, scales)` for the local slice, or for the
    whole batch if `gather=True`.  With `get_Wx=False`, `Wx` is None: it is neither
    computed into memory on the fused route nor gathered, which halves the gather.
    `_compute` (tests) replaces the transform."""
    if x.ndim != 2:
        raise ValueError("sharded execution needs a batched input [B, N]; a single "
                         "signal does not shard (one global FFT): run replicas")
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    B = x.shape[0]
    lo, hi = shard_bounds(B, rank, world)
    if _compute is None:
        from ._ssq_cwt import ssq_cwt as _compute
    if not get_Wx:
        kw['get_Wx'] = False
    if hi > lo:
        Tx, Wx, ssq_freqs, scales = _compute(x[lo:hi], *args, **kw)[:4]
    else:                                   # more ranks than signals
        Tx1, Wx1, ssq_freqs, scales = _compute(x[:1], *args, **kw)[:4]
        Tx, Wx = Tx1[:0], (None if Wx1 is None else Wx1[:0])
    if gather and world > 1:
        Tx = gather_batch(Tx, B, group)
        Wx = None if Wx is None else gather_batch(Wx, B, group)
    return Tx, Wx, ssq_freqs, scales
