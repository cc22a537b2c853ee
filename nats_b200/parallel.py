"""Data parallelism of the hot path (SURVEY 8(e)): the batch dimension shards across ranks (one process per GPU),
parameters and optimiser state are replicated, and ONE all-reduce per step sums the flat gradient buffer -- whose
tail slot carries the cost, so no second collective is needed.  Every rank scales its local gradient by
1 / (global batch), hence the sum equals d mean(cost) of nats.py:1323; clipping (nats.py:1344-1353) and the
optimiser then see identical buffers on all ranks.  Backend-agnostic (NCCL on GPUs, gloo in the CPU tests)."""


def world():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def grad_scale(local_batch, world_size, global_batch=None):
    """weight of every local sample's cost so that the all-reduced sum is the mean over the global batch"""
    return 1.0 / float(global_batch if global_batch is not None else local_batch * world_size)


def shard(seqs_x, seqs_y, rank, world_size):
    """contiguous, equal shards of a global batch of sentence pairs (the last ranks may get one pair less)"""
    n = len(seqs_x)
    per = (n + world_size - 1) // world_size
    lo, hi = min(rank * per, n), min((rank + 1) * per, n)
    return seqs_x[lo:hi], seqs_y[lo:hi]


def allreduce_flat(flat, async_op=False, group=None):
    """in-place SUM of (a slice of) the flat gradient buffer over all ranks; no-op for a single process.
    async_op: returns the work handle (wait() orders the current stream after the collective)."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        w = dist.all_reduce(flat, op=dist.ReduceOp.SUM, async_op=async_op, group=group)
        return w if async_op else flat
    return None if async_op else flat


def side_group(max_ctas=4):
    """A second NCCL communicator limited to `max_ctas` CTAs, for the all-reduce that runs UNDER the persistent encoder-
    backward kernel: that kernel holds 128 of the 132 SMs for milliseconds, a collective asking for more CTAs than the SMs left
    would simply wait for it to finish.  None when not applicable (single process, gloo, old torch)."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
        return None
    if dist.get_backend() != 'nccl':
        return None
    try:
        opts = dist.ProcessGroupNCCL.Options()
        opts.config.max_ctas = int(max_ctas)
        opts.config.min_ctas = 1
        return dist.new_group(backend='nccl', pg_options=opts)
    except Exception:
        return None


def shard_batch(seqs_x, seqs_y, rank, world_size):
    """What one rank trains on out of a GLOBAL batch read by every rank (train() of nats.py:1384-1411, made data
    parallel): contiguous shards of the pairs; prepare_data cuts long pairs instead of dropping them (nats.py:210-223), so
    the divisor of the mean cost (nats.py:1323) is the number of pairs of the global batch, known to every rank.
    Returns (x_shard, y_shard, n_global); a shard may be empty (then that rank only contributes zeros)."""
    n = len(seqs_x)
    sx, sy = shard(seqs_x, seqs_y, rank, world_size)
    return sx, sy, n
