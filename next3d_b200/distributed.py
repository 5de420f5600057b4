"""Multi-GPU plumbing for the one place the hot path shards: independent (latent, camera, mesh) samples.

One process per GPU (torchrun), contiguous split of the sample list across ranks, no data-path collective inside the
generator; a single gather of the output images to rank 0 (NCCL over NVLink on GPUs, gloo in the CPU tests) that can be
issued on a side stream so it overlaps the next micro-batch (SURVEY.md section 8e).
"""
import os

import torch
import torch.distributed as dist


def init_from_env(backend=None):
    """Initialise torch.distributed from torchrun's environment; returns (rank, world, local_rank). No-op for world 1."""
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    if world > 1 and not dist.is_initialized():
        # NCCL writes its debug output (the version banner included, at any NCCL_DEBUG level) to STDOUT unless told otherwise:
        # send it to stderr so that a caller's stdout stays machine-readable (bench.py prints one JSON line)
        os.environ.setdefault('NCCL_DEBUG_FILE', '/dev/stderr')
        backend = backend or ('nccl' if torch.cuda.is_available() else 'gloo')
        os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
        if backend == 'nccl':
            torch.cuda.set_device(local)
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    return rank, world, local


def shard_range(total, rank, world):
    """Contiguous [start, stop) of `total` samples owned by `rank` (first `total % world` ranks get one extra)."""
    base, extra = divmod(total, world)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


def gather_images(local_images, dst=0, sizes=None):
    """Gather per-rank image batches to `dst`: returns [sum(B_r), ...] on dst (rank order), None elsewhere.  `sizes`: batch size of
    every rank when the shards are unequal (shard_range with total % world != 0) -- smaller shards are padded to the largest for
    the collective and trimmed on dst; None = all ranks hold the same number of images."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return local_images
    world, rank = dist.get_world_size(), dist.get_rank()
    bmax = local_images.shape[0] if sizes is None else max(sizes)
    send = local_images.contiguous()
    if send.shape[0] < bmax:
        send = torch.cat([send, send.new_zeros((bmax - send.shape[0],) + tuple(send.shape[1:]))], 0)
    if rank == dst:
        out = torch.empty((world,) + tuple(send.shape), dtype=send.dtype, device=send.device)
        dist.gather(send, list(out.unbind(0)), dst=dst)
        if sizes is None:
            return out.flatten(0, 1)
        return torch.cat([out[r, :sizes[r]] for r in range(world)], 0)
    dist.gather(send, None, dst=dst)
    return None


def max_over_ranks(value, device):
    """Scalar max over ranks (device timing of multi-GPU runs is the slowest rank's)."""
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item()


class RankError(RuntimeError):
    """A failure on one of the ranks, raised on every rank: `rank` is the first failing rank, `message` its error."""

    def __init__(self, rank, message):
        super().__init__(f'rank {rank} failed: {message}')
        self.rank, self.message = rank, message


def rank_world(group=None):
    """(rank, world) in `group` (None = the default group); (0, 1) when torch.distributed is not initialised."""
    if not dist.is_initialized():
        return 0, 1
    return dist.get_rank(group), dist.get_world_size(group)


def agree(error, group=None):
    """Every rank passes its error message or None; raises RankError on every rank if any rank passed one (the first failing
    rank's), so that all ranks leave together instead of waiting for a rank that has gone.  No-op in one process."""
    if rank_world(group)[1] == 1:
        return
    errors = [None] * dist.get_world_size(group)
    dist.all_gather_object(errors, error, group=group)
    for r, e in enumerate(errors):
        if e is not None:
            raise RankError(r, e)


def run_together(body, group=None):
    """Run body() on this rank, then agree: in one process an exception of body() propagates unchanged; under torch.distributed a
    failure becomes this rank's message, and every rank raises RankError once all of them have finished body()."""
    err = None
    try:
        body()
    except Exception as e:
        if rank_world(group)[1] == 1:
            raise
        err = f'{type(e).__name__}: {e}'
    agree(err, group)


def gather_to_root(obj, group=None):
    """The picklable `obj` of every rank, in rank order, on rank 0 of `group` (host memory: meant for a gloo group); None on the
    other ranks.  In one process: [obj]."""
    rank, world = rank_world(group)
    if world == 1:
        return [obj]
    out = [None] * world if rank == 0 else None
    dist.gather_object(obj, out, dst=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
    return out
