"""Batched Chamfer over independent (x_b, y_b) pairs, and its multi-GPU form.

Pairs are independent, so the multi-GPU scheme is pure data parallelism (SURVEY.md 8e): each rank
(one process per GPU, `torch.distributed`) runs the single-GPU batched path on its contiguous shard
of pairs and the only traffic is one all-reduce of a single fp64 (the batch sum) -- or one
all-gather of the per-pair values when the caller wants them all.
"""
import numpy as _np

from . import _pcu_internal
from ._call import _as_form, _asarrays, _call_args, _dtype_name, _form, _numpy, _torch


def batched_chamfer(x, y, max_points_per_leaf=10, return_sum=False, device=-1):
    """x: (B, n, 3), y: (B, m, 3) float32, numpy or CUDA tensors -> (B,) Chamfer distances
    (and, with return_sum, their fp64 sum as computed on the device)."""
    arrays = _asarrays([x, y])
    form = _form(arrays, ["x", "y"])
    x, y = arrays
    if _dtype_name(x) != "float32" or _dtype_name(y) != "float32":
        raise ValueError("batched_chamfer_distance: x and y must both be float32")
    if len(x.shape) != 3 or len(y.shape) != 3 or x.shape[2] != 3 or y.shape[2] != 3 or x.shape[0] != y.shape[0]:
        raise ValueError("batched_chamfer_distance: x and y must have shape (B, n, 3) and (B, m, 3)")
    if x.shape[0] == 0 or x.shape[1] == 0 or y.shape[1] == 0:
        raise ValueError("Invalid input set with zero elements: x and y must have shape (B, n, 3) and (B, m, 3)")
    if form != "cuda":
        out, total = _pcu_internal._batched_chamfer_host(*_numpy([x, y]), int(max_points_per_leaf), int(device))
        out = _as_form(form, out)
        return (out, total) if return_sum else out
    torch = _torch()
    xs, ys = x.detach().contiguous(), y.detach().contiguous()
    B = xs.shape[0]
    out = torch.empty(B, dtype=torch.float32, device=xs.device)
    total = torch.empty((), dtype=torch.float64, device=xs.device)   # written by the last kernel of the call
    _pcu_internal._batched_chamfer_device(xs.data_ptr(), ys.data_ptr(), B, xs.shape[1], ys.shape[1], out.data_ptr(),
                                          total.data_ptr() if return_sum else 0, int(max_points_per_leaf), *_call_args(xs))
    return (out, total) if return_sum else out


def shard_bounds(batch, world_size, rank):
    """Contiguous block of pairs owned by `rank` (sizes differ by at most one)."""
    base, extra = divmod(int(batch), int(world_size))
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def reduce_sum(local, group=None):
    """All-reduce (sum) of one fp64 scalar per rank: the only exchange of the sharded batched path."""
    torch = _torch()
    import torch.distributed as dist
    if not isinstance(local, torch.Tensor):
        local = torch.tensor(float(local), dtype=torch.float64)
    local = local.to(torch.float64).reshape(1).clone()
    if dist.is_available() and dist.is_initialized():
        dist.all_reduce(local, op=dist.ReduceOp.SUM, group=group)
    return local.reshape(())


class ScalarSumExchange:
    """The path's only exchange -- the sum over ranks of one fp64 per rank -- kept OFF the caller's stream.

    `submit(t)` orders a side stream behind the caller's current stream (one event, no host wait) and
    all-reduces the contiguous fp64 tensor `t` in place there, so the collective of step s runs while the
    caller's stream is already binning step s + 1; `wait()` makes the caller's stream wait for everything
    submitted so far and returns the last tensor (now the sum over all ranks).  Without an initialised process
    group both are no-ops."""

    def __init__(self, device, group=None):
        torch = _torch()
        import torch.distributed as dist
        self._dist = dist if (dist.is_available() and dist.is_initialized()) else None
        self.group = group
        self.device = torch.device(device)
        self.stream = torch.cuda.Stream(device=self.device) if self._dist is not None else None
        self.event = torch.cuda.Event() if self._dist is not None else None
        self.last = None

    def submit(self, t):
        torch = _torch()
        if t.dtype != torch.float64 or not t.is_contiguous():
            raise ValueError("ScalarSumExchange.submit wants a contiguous float64 tensor")
        self.last = t
        if self._dist is None:
            return t
        self.event.record(torch.cuda.current_stream(self.device))
        self.stream.wait_event(self.event)
        with torch.cuda.stream(self.stream):
            self._dist.all_reduce(t, op=self._dist.ReduceOp.SUM, group=self.group)
        t.record_stream(self.stream)
        return t

    def wait(self):
        if self._dist is not None:
            _torch().cuda.current_stream(self.device).wait_stream(self.stream)
        return self.last


def distributed_chamfer_sum(x, y, exchange, max_points_per_leaf=10):
    """One (x, y) pair per rank (CUDA tensors): the fused bidirectional sweep of this rank's pair, whose last CTA
    leaves the pair's Chamfer value in fp64 in the statistics record (pcu_b200_nn_stats.pair_value), followed by
    the sum over ranks of that one fp64 on `exchange`'s side stream.  Returns the 1-element fp64 tensor that
    holds the all-rank sum once `exchange.wait()` has been called; no torch kernel and no host synchronisation
    sit between the sweep and the collective."""
    from . import _pair_value, _sweep
    form, _, words, _, _ = _sweep(x, y, True, max_points_per_leaf, None)
    if form != "cuda":
        raise ValueError("distributed_chamfer_sum wants CUDA tensors")
    return exchange.submit(_pair_value(words))


def gather_values(vals, batch, group=None):
    """All-gather of the per-pair values of every rank's shard (see shard_bounds) into the (batch,) vector."""
    torch = _torch()
    import torch.distributed as dist
    if not isinstance(vals, torch.Tensor):
        vals = torch.from_numpy(_np.asarray(vals))
    if not (dist.is_available() and dist.is_initialized()):
        return vals
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    lo, hi = shard_bounds(batch, world, rank)
    if vals.numel() != hi - lo:
        raise ValueError("rank %d owns pairs [%d, %d) but passed %d values" % (rank, lo, hi, vals.numel()))
    width = (int(batch) + world - 1) // world
    padded = torch.zeros(width, dtype=vals.dtype, device=vals.device)
    padded[: vals.numel()] = vals
    gathered = [torch.empty_like(padded) for _ in range(world)]
    dist.all_gather(gathered, padded, group=group)
    parts = []
    for r in range(world):
        rlo, rhi = shard_bounds(batch, world, r)
        parts.append(gathered[r][: rhi - rlo])
    return torch.cat(parts)


def distributed_batched_chamfer_sum(x_shard, y_shard, group=None, max_points_per_leaf=10):
    """Every rank passes ITS shard of pairs; returns the fp64 sum of the Chamfer distances of all
    pairs of all ranks (a 0-dim tensor on the shard's device).  One all-reduce of one scalar."""
    _, local = batched_chamfer(x_shard, y_shard, max_points_per_leaf, return_sum=True)
    return reduce_sum(local, group)


def distributed_batched_chamfer(x_shard, y_shard, batch, group=None, max_points_per_leaf=10):
    """Every rank passes its shard (see shard_bounds); returns the (batch,) per-pair values on every
    rank.  One all-gather of at most ceil(batch / world) floats per rank."""
    return gather_values(batched_chamfer(x_shard, y_shard, max_points_per_leaf), batch, group)
