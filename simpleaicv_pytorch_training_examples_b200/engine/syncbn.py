"""Synchronized BatchNorm across data-parallel ranks (nn.SyncBatchNorm's semantics, the reference's ``sync_bn``).

Every BatchNorm of the conv runtimes computes per-channel sums into a small fp32 buffer before it applies them; the
exchange sits between the two steps:

  forward   the partial sums are folded into stats [2C + 2] (sum | sum of squares | row count in two exact parts,
            ops.bn_stats_fold), all-reduced, and finalized with the global row count (ops.bn_finalize_folded): mean,
            variance and the running statistics (unbiased over the global count) are the same on every rank.
  backward  a copy of the reduced sums (sum dy | sum dy * xhat) is all-reduced: dx uses the global sums over the
            global count, dgamma / dbeta the local sums (the data-parallel wrapper averages them like every other
            gradient).

The exchanges run on the compute stream, in the order the layers run, over the group handed to the runtime
(``RuntimeModule.set_bn_group``).  That group must be dedicated to them: the data-parallel wrapper all-reduces gradient
buckets from a side stream during the backward, and two streams issuing collectives on one communicator could order
them differently on different ranks.  In eval, or with a group of one rank, nothing is exchanged and the arithmetic is
that of the unsynchronized BatchNorm, bit for bit.
"""
import contextlib

import torch.distributed as dist

from .. import ops

_GROUP = None   # the group of the runtime forward / backward being run, None when BatchNorm is not synchronized


@contextlib.contextmanager
def exchanging(group):
    """Inside, training-mode BatchNorm layers synchronize over `group` (None or a group of one rank: they do not)."""
    global _GROUP
    if group is not None and dist.get_world_size(group) <= 1:
        group = None
    old, _GROUP = _GROUP, group
    try:
        yield
    finally:
        _GROUP = old


def finalize(partials, partial_rows, rows, gamma, beta, rmean, rvar, scale_shift, saved, eps, momentum):
    """ops.bn_finalize over this rank's statistics, or over every rank's when synchronized.  Returns the exchanged
    statistics buffer (its row count is the backward's) or None."""
    if _GROUP is None:
        ops.bn_finalize(partials, gamma, beta, rmean, rvar, scale_shift, saved, rows, eps, momentum,
                        partial_rows=partial_rows)
        return None
    stats = ops.bn_stats_fold(partials, rows, gamma.numel(), partial_rows=partial_rows)
    dist.all_reduce(stats, group=_GROUP)
    ops.bn_finalize_folded(stats, gamma, beta, rmean, rvar, scale_shift, saved, eps, momentum)
    return stats


def backward_sums(sums, stats, c):
    """The backward sums of a BatchNorm whose forward returned `stats` from finalize(), and the keyword arguments of
    the apply kernels: (sums, {}) unsynchronized; else (sums reduced over ranks, {local_sums, count})."""
    if stats is None:
        return sums, {}
    if _GROUP is None:
        raise RuntimeError('the backward of a synchronized BatchNorm forward must run with its exchange group')
    total = sums.clone()
    dist.all_reduce(total, group=_GROUP)
    return total, {'local_sums': sums, 'count': ops.bn_sync_count(stats, c)}
