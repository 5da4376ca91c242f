"""Data parallelism for the training step: the only multi-GPU mechanism on the path (reference trainer.py:78-82 wraps
the model in DistributedDataParallel; SURVEY.md §8e).

One process per GPU, full replica each, rank r draws its own batch; once per step the gradients are averaged over
NVLink/NVSwitch.  Two mechanisms:
  * `FlatGradAverager`: ONE flat all-reduce after backward (any model);
  * `OverlappedGradAverager`: the fused ImageGPT stack produces every gradient inside a single autograd node, so DDP's
    per-parameter hooks have nothing to overlap with; instead the stack itself hands each transformer block's weight
    gradients (one contiguous slice of its gradient arena, 12.6 MB at C5) to `bucket_hook` the moment the block's last
    wgrad GEMM is queued.  The hook launches an asynchronous all-reduce (NCCL's own stream, ordered after the kernels
    queued so far), the backward of the next block runs underneath it, and the stack waits for all buckets before it
    returns -- the reference's "bucketed all-reduce overlapped with backward" (trainer.py:78-82) at block granularity.
    The few small gradients outside the arena (biases, LayerNorm, embeddings) go through one flat all-reduce afterwards.
The helpers are backend-agnostic (`gloo` on CPU in the tests).
"""

import os

import torch
import torch.distributed as dist

# SMs the persistent GEMM / attention grids leave to the NCCL kernels of the in-backward bucket all-reduces (world > 1).
# Both knobs default to "off" (PG_DP_RESERVE_SMS, PG_NCCL_MAX_CTAS).
DEFAULT_RESERVED_SMS = 0

# CTAs NCCL may use per collective (0 = NCCL's own choice).
DEFAULT_NCCL_MAX_CTAS = 0


def configure_nccl():
    """Call before `init_process_group`: caps NCCL's CTAs per collective (NCCL_MAX_CTAS; PG_NCCL_MAX_CTAS overrides, 0 keeps
    NCCL's default)."""
    n = int(os.environ.get("PG_NCCL_MAX_CTAS", str(DEFAULT_NCCL_MAX_CTAS)))
    if n > 0:
        os.environ.setdefault("NCCL_MAX_CTAS", str(n))
        os.environ.setdefault("NCCL_MIN_CTAS", "1")


def broadcast_parameters(module, src=0):
    """Makes every rank start from rank `src`'s parameters and buffers (what DDP does at construction)."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return
    with torch.no_grad():
        for t in list(module.parameters()) + list(module.buffers()):
            dist.broadcast(t.data, src=src)
            torch.autograd.graph.increment_version(t)  # written through .data: its bf16 copies are stale


class FlatGradAverager:
    """Averages the gradients of `params` across ranks with one all-reduce over a persistent flat fp32 bucket."""

    def __init__(self, params):
        self.params = [p for p in params if p.requires_grad]
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        numel = sum(p.numel() for p in self.params)
        dev = self.params[0].device if self.params else torch.device("cpu")
        self.flat = torch.zeros(numel, dtype=torch.float32, device=dev)
        self.views, off = [], 0
        for p in self.params:
            self.views.append(self.flat[off: off + p.numel()].view_as(p))
            off += p.numel()

    @torch.no_grad()
    def average_(self):
        """In place: p.grad <- mean over ranks of p.grad (parameters without a gradient contribute zeros).

        Packing and unpacking are multi-tensor copies (a few launches for the whole bucket, not two per parameter);
        NCCL averages inside the collective, other backends sum and the bucket is scaled afterwards."""
        if self.world == 1:
            return
        have = [(p, v) for p, v in zip(self.params, self.views) if p.grad is not None]
        for p, v in zip(self.params, self.views):
            if p.grad is None:
                v.zero_()
        if have:
            torch._foreach_copy_([v for _, v in have], [p.grad for p, _ in have])
        if dist.get_backend() == "nccl":
            dist.all_reduce(self.flat, op=dist.ReduceOp.AVG)
        else:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM)
            self.flat.div_(self.world)
        if have:
            torch._foreach_copy_([p.grad for p, _ in have], [v for _, v in have])
        for p, v in zip(self.params, self.views):
            if p.grad is None:
                p.grad = v.clone()


class _PendingBucket:
    """Handle of one in-flight bucket: wait() orders the current stream after the collective (and applies the 1/world
    scale for backends that cannot average inside the collective)."""

    def __init__(self, work, flat, scale):
        self.work, self.flat, self.scale = work, flat, scale

    def wait(self):
        self.work.wait()
        if self.scale is not None:
            self.flat.mul_(self.scale)


def bucket_all_reduce_mean(flat):
    """Asynchronous in-place mean over ranks of a contiguous gradient bucket; returns a handle with wait()."""
    world = dist.get_world_size()
    if dist.get_backend() == "nccl":
        return _PendingBucket(dist.all_reduce(flat, op=dist.ReduceOp.AVG, async_op=True), flat, None)
    return _PendingBucket(dist.all_reduce(flat, op=dist.ReduceOp.SUM, async_op=True), flat, 1.0 / world)


class OverlappedGradAverager:
    """Block-bucketed gradient averaging overlapped with backward for models that expose
    `set_grad_bucket_hook(fn)` / `bucketed_parameters()` (the fused ImageGPT stack); everything else (and every other
    model) falls back to the flat bucket."""

    def __init__(self, model, params=None):
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        params = list(model.parameters()) if params is None else list(params)
        bucketed = []
        self._model = model
        if self.world > 1 and hasattr(model, "set_grad_bucket_hook"):
            model.set_grad_bucket_hook(bucket_all_reduce_mean)
            bucketed = list(model.bucketed_parameters())
            reserve = int(os.environ.get("PG_DP_RESERVE_SMS", str(DEFAULT_RESERVED_SMS)))
            if bucketed and reserve > 0 and torch.cuda.is_available():
                from . import _lib

                _lib.reserve_sms(reserve)  # the bucket all-reduces run next to the backward GEMMs (see pg_reserve_sms)
        skip = {id(p) for p in bucketed}
        self.n_bucketed = len(bucketed)
        self.rest = FlatGradAverager([p for p in params if id(p) not in skip])

    def average_(self):
        """Call after backward: the arena-backed gradients were averaged inside backward already."""
        self.rest.average_()

    def close(self):
        """Detaches the bucket hook from the model (its backward then issues no collective any more)."""
        if self.n_bucketed and hasattr(self._model, "set_grad_bucket_hook"):
            self._model.set_grad_bucket_hook(None)


def shard_seed(base_seed, rank):
    """Synthetic-data seed of a rank: every rank draws its own batch (weak scaling, like the reference's loaders)."""
    return int(base_seed) + int(rank)


def shard_samples(n_samples, rank, world):
    """`sample()` across GPUs is replicas only (SURVEY.md §8e): rank r draws its share of the `n_samples` images, no
    communication.  Returns the number of images rank `rank` generates (shares differ by at most one)."""
    base, extra = divmod(int(n_samples), int(world))
    return base + (1 if rank < extra else 0)
