"""gem_b200/dist.py -- host-side sharding rules of the multi-GPU path (one process per GPU).

The same formulas are used inside libgemb200 (core.cu::gemb_graph_upload, n2v.cu::gemb_node2vec);
keeping them here lets the CPU test-suite check them with gloo (tests/test_dist_cpu.py)."""
import os

import numpy as np


def rows_per_rank(n, nranks):
    """Equal row shards (the all-gather needs equal counts): ceil(n / P); the tail is zero padding."""
    return (n + nranks - 1) // nranks


def row_range(n, rank, nranks):
    per = rows_per_rank(n, nranks)
    r0 = min(n, rank * per)
    return r0, min(n, r0 + per)


def walk_range(total_walks, rank, nranks):
    """Contiguous share of the num_walks*N walk index space (walk w = round*N + position)."""
    per = (total_walks + nranks - 1) // nranks
    w0 = min(total_walks, per * rank)
    return w0, min(total_walks, w0 + per)


def pad_rows(X, n_shard):
    """Row shard -> n_shard rows (zero padded), what every rank contributes to the all-gather."""
    out = np.zeros((n_shard,) + X.shape[1:], dtype=X.dtype)
    out[:X.shape[0]] = X
    return out


def spmd(device=None):
    """(torch.distributed module, rank, world, device) of this process.  world > 1 only under an initialised process
    group; the device is the given one, else LOCAL_RANK when world > 1, else 0."""
    dist_mod, rank, world = None, 0, 1
    if int(os.environ.get('WORLD_SIZE', '1')) > 1:
        try:
            import torch.distributed as td
        except ImportError:
            td = None
        if td is not None and td.is_available() and td.is_initialized():
            dist_mod, rank, world = td, td.get_rank(), td.get_world_size()
    if device is None:
        device = int(os.environ.get('LOCAL_RANK', '0')) if world > 1 else 0
    return dist_mod, rank, world, device


def init_comm_from_torch(ctx, dist_module, rank, world):
    """Bootstrap the library's NCCL communicator through an already initialised torch.distributed group."""
    from gem_b200 import _native
    uid = [_native.comm_unique_id() if rank == 0 else None]
    dist_module.broadcast_object_list(uid, src=0)
    ctx.comm_init(rank, world, uid[0])


def halo_plan(n, row0, n_shard, indices):
    """Host-side statement of gem_b200/csrc/halo.cu::halo_build for one rank (NumPy; the library does the same on the
    device with cub): H = the sorted distinct REMOTE columns the shard references; indices_ext = the column ids with
    local columns renumbered to [0, n_shard) and remote ones to n_shard + (position in H)."""
    indices = np.asarray(indices, dtype=np.int64)
    lo, hi = row0, min(row0 + n_shard, n)
    remote = (indices < lo) | (indices >= hi)
    H = np.unique(indices[remote])
    ext = np.where(remote, n_shard + np.searchsorted(H, indices), indices - lo)
    return H.astype(np.int32), ext.astype(np.int32)


def push_lists(H_all, row0, n_shard, n, rank):
    """Who needs my rows: for every peer q the slots of H_q that fall into [row0, row0 + n_shard) -> (local row, q, slot)."""
    lo, hi = row0, min(row0 + n_shard, n)
    out = []
    for q, H in enumerate(H_all):
        if q == rank:
            continue
        a, b = np.searchsorted(H, lo), np.searchsorted(H, hi)
        for slot in range(a, b):
            out.append((int(H[slot]) - lo, q, slot))
    return out
