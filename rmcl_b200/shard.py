"""Partitioning of independent units (particles / poses) across ranks -- SURVEY.md section 8e.

No arithmetic crosses particles or poses on this path (PCDSensorUpdaterEmbree.cpp:330-341), so multi-GPU is a contiguous
split with the map replicated per GPU and NO data-path collective; the only exchange is gathering the shards' results.
The stages of the particle-filter cycle with a real exchange are resampling (opponents are drawn from ALL particles,
resampling.cu:137): `gladiator_resample_sharded` all-gathers the particle set first; and the Stein steps (every particle moves against a
reference set drawn from all particles, with a bandwidth from the whole set): `stein_update_sharded` all-gathers the poses and the
references' snapshot every iteration.
"""
from __future__ import annotations

import numpy as np


def shard_range(n: int, rank: int, world: int):
    """Contiguous [begin, end) of unit `rank` of `world`; sizes differ by at most one."""
    base, rem = divmod(n, world)
    begin = rank * base + min(rank, rem)
    return begin, begin + base + (1 if rank < rem else 0)


def gather_records(local: np.ndarray, dist, dst: int = 0):
    """Gather a structured numpy array (any record dtype) from all ranks onto `dst` with torch.distributed (gloo or nccl)."""
    import torch
    world, rank = dist.get_world_size(), dist.get_rank()
    raw = np.ascontiguousarray(local).view(np.uint8).reshape(-1)
    sizes = [torch.zeros(1, dtype=torch.int64) for _ in range(world)]
    dist.all_gather(sizes, torch.tensor([raw.size], dtype=torch.int64))
    m = int(max(s.item() for s in sizes))
    buf = torch.zeros(m, dtype=torch.uint8)
    buf[: raw.size] = torch.from_numpy(raw.copy())
    outs = [torch.zeros(m, dtype=torch.uint8) for _ in range(world)] if rank == dst else None
    dist.gather(buf, outs, dst=dst)
    if rank != dst:
        return None
    parts = [outs[r][: int(sizes[r].item())].numpy().view(local.dtype) for r in range(world)]
    return np.concatenate(parts)


def gladiator_resample_sharded(resample_fn, poses_local, attrs_local, dist, sync=None):
    """Gladiator resampling with particles sharded over ranks in equal contiguous slices (rank order = global order).

    poses_local (n, 8) / attrs_local (n, 9): float32 torch tensors (CUDA with nccl, CPU with gloo).  All-gathers the particle set
    (68 B per particle -- the exchange step), then calls `resample_fn(P_all, A_all, first, n_local) -> (P_new, A_new)` for this rank's
    champions.  The draws are keyed by the global particle index, so the concatenation over ranks equals the unsharded result."""
    import torch
    ws, rank = dist.get_world_size(), dist.get_rank()
    n_local = poses_local.shape[0]
    counts = torch.zeros(ws, dtype=torch.int64, device=poses_local.device)
    counts[rank] = n_local
    dist.all_reduce(counts)
    counts = [int(c) for c in counts.tolist()]
    if len(set(counts)) != 1:
        raise ValueError(f"gladiator_resample_sharded needs equal shard sizes, got {counts}")
    if sync is not None:
        sync()                      # whatever produced the local particles (on the handle's stream) must be complete before the collective reads them
    P_all = torch.empty((ws * n_local, 8), dtype=torch.float32, device=poses_local.device)
    A_all = torch.empty((ws * n_local, 9), dtype=torch.float32, device=poses_local.device)
    dist.all_gather_into_tensor(P_all, poses_local.contiguous())
    dist.all_gather_into_tensor(A_all, attrs_local.contiguous())
    if sync is not None:
        sync()                      # the collective ran on torch's stream; the resampling kernel runs on the handle's
    return resample_fn(P_all, A_all, rank * n_local, n_local)


def stein_update_sharded(begin_fn, score_fn, move_fn, result_fn, poses_local, dist, iterations: int, n_ref: int):
    """Stein variational steps (b2_pf_stein_slice_*, SURVEY L14) on a particle set sharded over ranks in equal contiguous slices (rank
    order = global order); poses_local, an (n, 8) float32 torch tensor (CUDA with nccl, CPU with gloo), is moved in place.

    Each rank scores the range shard_range(m, rank, world) of the m references of J and moves its own slice.  Per iteration k: all-gather
    the poses (32 B per particle), `score_fn(P_all, k, snap)` into this rank's (j_count, 6) float32 rows of the snapshot, all-gather the
    snapshots (24 B per reference, padded to equal length), `move_fn(P_all, snap_all, k, poses_local)`.  `begin_fn(n_all, first, n_local,
    j_first, j_count)` opens the session first; `result_fn()` -> dict(bandwidth, n_ref, n_blocked, n_steps, sum_step_t2, sum_step_r2)
    reads this rank's record at the end.  The slices then equal the unsharded steps of the whole set byte for byte.
    -> the whole set's record dict(bandwidth, n_ref, n_blocked, rms_step_t, rms_step_r): n_blocked, n_steps and the two sums all-reduced."""
    import torch
    ws, rank = dist.get_world_size(), dist.get_rank()
    n_local = poses_local.shape[0]
    dev = poses_local.device
    counts = torch.zeros(ws, dtype=torch.int64, device=dev)
    counts[rank] = n_local
    dist.all_reduce(counts)
    counts = [int(c) for c in counts.tolist()]
    if len(set(counts)) != 1:
        raise ValueError(f"stein_update_sharded needs equal shard sizes, got {counts}")
    n_all = ws * n_local
    m = n_all if n_ref == 0 or n_ref >= n_all else n_ref
    j_first, j_end = shard_range(m, rank, ws)
    j_len = -(-m // ws)                         # the longest range; the others are padded to it for all_gather_into_tensor
    ranges = [shard_range(m, r, ws) for r in range(ws)]
    pick = torch.tensor([r * j_len + i for r, (a, b) in enumerate(ranges) for i in range(b - a)], dtype=torch.int64, device=dev)
    begin_fn(n_all, rank * n_local, n_local, j_first, j_end - j_first)
    P_all = torch.empty((n_all, 8), dtype=torch.float32, device=dev)
    snap = torch.zeros((j_len, 6), dtype=torch.float32, device=dev)
    snap_gathered = torch.empty((ws * j_len, 6), dtype=torch.float32, device=dev)
    snap_all = torch.empty((m, 6), dtype=torch.float32, device=dev)
    for k in range(iterations if n_all else 0):
        dist.all_gather_into_tensor(P_all, poses_local)
        score_fn(P_all, k, snap)
        dist.all_gather_into_tensor(snap_gathered, snap)
        torch.index_select(snap_gathered, 0, pick, out=snap_all)
        move_fn(P_all, snap_all, k, poses_local)
    r = result_fn()
    sums = torch.tensor([float(r["n_blocked"]), float(r["n_steps"]), r["sum_step_t2"], r["sum_step_r2"]], dtype=torch.float64, device=dev)
    dist.all_reduce(sums)
    n_blocked, n_steps, t2, r2 = sums.tolist()
    rms = lambda s: float(np.float32(np.sqrt(s / n_steps))) if n_steps > 0 else 0.0
    return {"bandwidth": tuple(r["bandwidth"]), "n_ref": int(r["n_ref"]), "n_blocked": int(n_blocked), "rms_step_t": rms(t2), "rms_step_r": rms(r2)}
