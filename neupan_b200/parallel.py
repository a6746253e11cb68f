"""Multi-GPU plumbing of the hot path (SURVEY.md 8e): environments are independent, so the batch is
split into contiguous blocks, one process per GPU; the single exchange of a control step is the
gather of the packed per-environment result [S 3(T+1) | U 2T | D T | min_distance 1].

Works with any torch.distributed backend (NCCL over NVLink between GPUs, gloo in the CPU tests).
"""
from __future__ import annotations

import torch
import torch.distributed as dist


def shard_range(total_envs: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous block [lo, hi) of environments owned by `rank` (sizes differ by at most one)."""
    base, rem = divmod(total_envs, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def pack_results(S: torch.Tensor, U: torch.Tensor, D: torch.Tensor, min_distance: torch.Tensor) -> torch.Tensor:
    B = S.shape[0]
    return torch.cat([S.reshape(B, -1), U.reshape(B, -1), D.reshape(B, -1), min_distance.reshape(B, 1)], dim=1).contiguous()


def unpack_results(packed: torch.Tensor, T: int):
    B = packed.shape[0]
    a, b, c = 3 * (T + 1), 3 * (T + 1) + 2 * T, 3 * (T + 1) + 3 * T
    return packed[:, :a].reshape(B, 3, T + 1), packed[:, a:b].reshape(B, 2, T), packed[:, b:c].reshape(B, 1, T), packed[:, c]


def gather_results(packed: torch.Tensor, total_envs: int, group=None) -> torch.Tensor:
    """all_gather of the per-rank packed results into (total_envs, width), rank-major = env order.
    Ranks may own different numbers of envs (shard_range); shorter shards are padded for the collective."""
    world = dist.get_world_size(group)
    if world == 1:
        return packed
    sizes = [shard_range(total_envs, r, world) for r in range(world)]
    longest = max(hi - lo for lo, hi in sizes)
    buf = packed
    if packed.shape[0] < longest:
        buf = torch.zeros((longest, packed.shape[1]), dtype=packed.dtype, device=packed.device)
        buf[: packed.shape[0]] = packed
    out = torch.empty((world * longest, packed.shape[1]), dtype=packed.dtype, device=packed.device)
    dist.all_gather_into_tensor(out, buf, group=group)
    if all(hi - lo == longest for lo, hi in sizes):
        return out
    return torch.cat([out[r * longest: r * longest + (hi - lo)] for r, (lo, hi) in enumerate(sizes)], dim=0)


class ShardedPAN:
    """One control step of `total_envs` environments over all ranks of a process group: every rank runs the PAN
    hot path on its contiguous block (shard_range) and the packed results are exchanged with one all_gather --
    the only collective of the path (SURVEY.md 8e).  Inputs are this rank's block, either CUDA tensors
    (device-resident step) or pinned host tensors (end-to-end step: H2D copies, compute, gather, and a D2H copy of
    the gathered result, all inside this call).

        sp = ShardedPAN(pan, total_envs)
        packed = sp.step(nom_s, nom_u, ref_s, ref_us, points, velocities)   # (total_envs, 64) for T = 10
        S, U, D, min_distance = unpack_results(packed, pan.T)
    """

    def __init__(self, pan, total_envs: int, group=None):
        self.pan, self.total, self.group = pan, int(total_envs), group
        self.world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if self.world > 1 else 0
        self.lo, self.hi = shard_range(self.total, self.rank, self.world)
        self._host_out = None

    def step(self, nom_s, nom_u, ref_s, ref_us, points=None, velocities=None, num_points=None) -> torch.Tensor:
        pan = self.pan
        host = nom_s.device.type != "cuda"
        with torch.no_grad():  # sharded control is inference (the gather is not differentiable); tune parameters through PAN itself
            # host inputs: nb_pan_forward_h2d uploads them in env chunks on a copy stream, the first DUNE pass of a chunk starts when its
            # points have landed; the results stay on the device for the gather
            S, U, D = pan(nom_s, nom_u, ref_s, ref_us, points, velocities, num_points, device_out=host)
        B = S.shape[0]
        md = pan.min_distance if torch.is_tensor(pan.min_distance) else torch.full((B,), float("inf"), device=S.device)
        if D is None:
            D = torch.zeros((B, 1, pan.T), device=S.device)
        packed = pack_results(S, U, D, md)
        out = gather_results(packed, self.total, self.group) if self.world > 1 else packed
        if not host:
            return out
        if self._host_out is None or self._host_out.shape != out.shape:
            self._host_out = torch.empty(out.shape, dtype=out.dtype, pin_memory=True)
        self._host_out.copy_(out, non_blocking=True)
        torch.cuda.current_stream(pan.device).synchronize()
        return self._host_out
