"""Frame-batch sharding across the GPUs of one box (SURVEY.md 8e).

The per-pair forward does not shard; pairs do.  One process per GPU (torch.distributed, NCCL over
NVLink/NVSwitch on the GPU box, gloo in the CPU tests):
  * broadcast_arena : ONE broadcast of the net's contiguous parameter arena from rank 0
  * shard_bounds    : contiguous split of B pairs over the ranks (first ranks take the remainder)
  * gather_flows    : all ranks' (b_r, 2, H, W) flow fields -> (B, 2, H, W) in global pair order on EVERY rank
  * gather_flows_to_root : the same, delivered to one rank only (what a serving front end needs: 1/world of the
                      all-gather traffic, and issued on a side stream it overlaps the next step's forward)
  * allreduce_gradients : data-parallel TRAINING (BASELINE config 5): every rank runs the step on its own pairs, then ONE
                      all-reduce over the contiguous parameter-gradient arena (fn2_net_param_diff_arena) averages the
                      gradients -- the reference's P2PSync tree (src/caffe/parallel.cpp:271-380) as a single NVSwitch collective
No collective exists inside a pair.  The reference has no inference data parallelism at all (its P2PSync
is training-only, src/caffe/parallel.cpp:271-380).
"""
import torch
import torch.distributed as dist


class DevicePtr(object):
    """Zero-copy torch view of raw device memory (the C-ABI hands out plain pointers)."""

    def __init__(self, ptr, nfloats):
        self.__cuda_array_interface__ = {"shape": (int(nfloats),), "typestr": "<f4", "data": (int(ptr), False), "version": 2}


def arena_tensor(net):
    ptr, nbytes = net.param_arena()
    return torch.as_tensor(DevicePtr(ptr, nbytes // 4), device="cuda")


def shard_bounds(total, world, rank):
    base, rem = divmod(int(total), int(world))
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def broadcast_arena(arena, src=0):
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.broadcast(arena, src=src)
    return arena


def gather_flows(local, total):
    """local: (b_r, 2, H, W) on this rank.  Returns the (total, 2, H, W) tensor on every rank."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return local
    world = dist.get_world_size()
    sizes = [shard_bounds(total, world, r) for r in range(world)]
    if all(hi - lo == sizes[0][1] - sizes[0][0] for lo, hi in sizes):
        out = local.new_empty((total,) + tuple(local.shape[1:]))
        dist.all_gather_into_tensor(out, local.contiguous())
        return out
    # uneven shards: pad to the largest shard (collectives want equal sizes), trim afterwards
    mx = max(hi - lo for lo, hi in sizes)
    padded = local.new_zeros((mx,) + tuple(local.shape[1:]))
    padded[:local.shape[0]] = local
    out = local.new_empty((world * mx,) + tuple(local.shape[1:]))
    dist.all_gather_into_tensor(out, padded)
    return torch.cat([out[r * mx:r * mx + (hi - lo)] for r, (lo, hi) in enumerate(sizes)], 0)


def gather_flows_to_root(local, out=None, dst=0):
    """Equal shards: local (b, 2, H, W) of every rank -> out (world*b, 2, H, W) on rank `dst` only (None elsewhere).
    One grouped send/recv (ncclSend/ncclRecv) instead of an all-gather: rank dst receives (world-1)*b flow fields, the others
    send b and receive nothing.  Runs on the CURRENT stream's NCCL queue: call it under a side stream to overlap compute."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        if out is not None:
            out.copy_(local)
            return out
        return local
    world, rank = dist.get_world_size(), dist.get_rank()
    if rank == dst:
        if out is None:
            out = local.new_empty((world * local.shape[0],) + tuple(local.shape[1:]))
        dist.gather(local, list(out.chunk(world)), dst=dst)
        return out
    dist.gather(local, None, dst=dst)
    return None


def grad_arena_tensor(net, trainable_only=False):
    """The gradient arena as a torch view; trainable_only: just the part the backward pass writes (net.trainable_diff_span()),
    which is what a stage trained on frozen predecessors has to all-reduce."""
    ptr, nbytes = net.trainable_diff_span() if trainable_only else net.param_diff_arena()
    return torch.as_tensor(DevicePtr(ptr, nbytes // 4), device="cuda")


def allreduce_gradients(grads, average=True):
    """grads: the contiguous gradient arena (grad_arena_tensor(net), or any tensor in the CPU tests).  Sum over the ranks, divided
    by the world size when `average` (each rank normalised its loss by its own batch, l1loss_layer.cu:83-88)."""
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(grads, op=dist.ReduceOp.SUM)
        if average:
            grads.mul_(1.0 / dist.get_world_size())
    return grads
