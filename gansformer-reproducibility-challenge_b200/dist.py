"""Data-parallel plumbing: one process per GPU (torchrun), NCCL over NVLink/NVSwitch.

The generator shards by images (SURVEY 8e): every image is independent through the whole network, so inference
needs no collective.  The collectives of the system are in the G/D training step: the gradient all-reduce (reference:
dnnlib/tflib/optimizer.py -> nccl_ops.all_sum over in-process towers, upstream; not in the checkout) and, with adaptive
augmentation, one two-float sum of the ADA accumulators per step (``allreduce_sum``).
"""
from __future__ import annotations

import os
from typing import Iterable, Tuple

import torch
import torch.distributed as dist


def env_world() -> Tuple[int, int, int]:
    """(rank, world_size, local_rank) from the torchrun environment; (0, 1, 0) when launched plainly."""
    return int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))


def init_distributed(backend: str | None = None) -> Tuple[int, int, int]:
    rank, world, local = env_world()
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        kwargs = {}
        if backend == "nccl":
            torch.cuda.set_device(local)
            kwargs["device_id"] = torch.device("cuda", local)
        dist.init_process_group(backend=backend, rank=rank, world_size=world, **kwargs)
    return rank, world, local


def shard_bounds(total: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous [lo, hi) slice of `total` items owned by `rank` (sizes differ by at most one)."""
    base, rem = divmod(total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_batch(t: torch.Tensor, rank: int, world: int) -> torch.Tensor:
    """Rank's slice of a globally generated batch: the union over ranks is the 1-GPU batch bit for bit."""
    lo, hi = shard_bounds(t.shape[0], rank, world)
    return t[lo:hi]


def allreduce_gradients(params: Iterable[torch.nn.Parameter], world: int) -> float:
    """Average gradients across ranks through ONE flat fp32 buffer (one all-reduce per network per step), synchronously.
    The simple form (tests, one-off reductions); the training step uses ``GradBuckets`` (bucketed, overlapped, no copies).

    Returns the number of bytes reduced.  No-op (0) when world == 1."""
    if world <= 1:
        return 0.0
    grads = [p.grad for p in params if p.grad is not None]
    if not grads:
        return 0.0
    flat = torch.cat([g.reshape(-1) for g in grads])
    dist.all_reduce(flat, op=dist.ReduceOp.SUM)
    flat.div_(world)
    off = 0
    for g in grads:
        n = g.numel()
        g.copy_(flat[off:off + n].view_as(g))
        off += n
    return float(flat.numel() * flat.element_size())


class GradBuckets:
    """Bucketed gradient all-reduce overlapped with the backward pass (SURVEY row f2; reference: dnnlib/tflib/optimizer.py ->
    nccl_ops.all_sum, upstream).

    * The gradients of a network LIVE in one pre-flattened fp32 buffer: every ``p.grad`` is a view into it, laid out in reverse
      parameter order (the order backward produces them), so a bucket is a contiguous slice -- no ``cat``, no copy-back.
    * A post-accumulate hook per parameter counts its bucket down; when the last gradient of a bucket has landed the bucket's
      all-reduce is enqueued on a communication stream (after an event on the compute stream) and overlaps the rest of backward.
      NCCL averages in the collective (ReduceOp.AVG); gloo (CPU tests) sums and divides.
    * ``finish()`` makes the compute stream wait for the communication stream.  Everything is stream-ordered (no host sync), so
      the whole step -- hooks included -- can be captured into a CUDA graph.
    """

    def __init__(self, params: Iterable[torch.nn.Parameter], world: int, bucket_mb: float = 32.0):
        self.world = world
        self.params = [p for p in params if p.requires_grad or True]
        if not self.params:
            raise ValueError("GradBuckets: no parameters")
        dev = self.params[0].device
        order = list(reversed(self.params))
        total = sum(p.numel() for p in order)
        self.flat = torch.zeros(total, dtype=torch.float32, device=dev)
        self.buckets = []                 # (lo, hi) slices of self.flat
        self._bucket_of = {}
        self._pending0 = []
        lim = max(1, int(bucket_mb * (1 << 20) / 4))
        off, lo, count = 0, 0, 0
        for p in order:
            n = p.numel()
            p.grad = self.flat[off:off + n].view_as(p)
            self._bucket_of[id(p)] = len(self.buckets)
            off += n
            count += 1
            if off - lo >= lim:
                self.buckets.append((lo, off)); self._pending0.append(count); lo, count = off, 0
        if off > lo:
            self.buckets.append((lo, off)); self._pending0.append(count)
        self._pending = list(self._pending0)
        self._active = False
        self._cuda = dev.type == "cuda"
        self._comm = torch.cuda.Stream(device=dev) if self._cuda else None
        self.bytes_per_step = float(total * 4)
        self._handles = [p.register_post_accumulate_grad_hook(self._hook) for p in self.params]

    # -- step protocol: begin() before backward, finish() after it ------------------------------------------------
    def begin(self):
        """Zero the flat buffer (one memset instead of one per parameter) and arm the hooks."""
        self.flat.zero_()
        for p in self.params:             # re-attach views an optimizer / zero_grad(set_to_none=True) may have dropped
            if p.grad is None or p.grad.data_ptr() < self.flat.data_ptr() or p.grad.data_ptr() >= self.flat.data_ptr() + self.flat.numel() * 4:
                self._reattach()
                break
        self._pending = list(self._pending0)
        self._active = self.world > 1

    def _reattach(self):
        off = 0
        for p in reversed(self.params):
            n = p.numel()
            p.grad = self.flat[off:off + n].view_as(p)
            off += n

    def _hook(self, p):
        if not self._active:
            return
        b = self._bucket_of[id(p)]
        self._pending[b] -= 1
        if self._pending[b] == 0:
            self._reduce(b)

    def _reduce(self, b):
        lo, hi = self.buckets[b]
        chunk = self.flat[lo:hi]
        if self._cuda:
            cur = torch.cuda.current_stream(self.flat.device)
            self._comm.wait_stream(cur)                       # the bucket's gradients are complete on the compute stream
            with torch.cuda.stream(self._comm):
                dist.all_reduce(chunk, op=dist.ReduceOp.AVG)
        else:
            dist.all_reduce(chunk, op=dist.ReduceOp.SUM)
            chunk.div_(self.world)

    def finish(self) -> float:
        """Reduce what the hooks did not (parameters without a gradient this step), then join the communication stream."""
        if not self._active:
            return 0.0
        for b, left in enumerate(self._pending):
            if left > 0:
                self._reduce(b)
        self._active = False
        if self._cuda:
            torch.cuda.current_stream(self.flat.device).wait_stream(self._comm)
        return self.bytes_per_step


def allreduce_sum(t: torch.Tensor) -> None:
    """In-place sum of a small tensor over ranks on the current stream (capturable with NCCL): the ADA accumulators of the training
    step, so that every rank holds the same augmentation strength."""
    dist.all_reduce(t, op=dist.ReduceOp.SUM)


def max_over_ranks(value: float, device=None) -> float:
    if not (dist.is_available() and dist.is_initialized()):
        return value
    t = torch.tensor([value], dtype=torch.float64, device=device if device is not None else "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def barrier():
    if dist.is_available() and dist.is_initialized():
        dist.barrier()
