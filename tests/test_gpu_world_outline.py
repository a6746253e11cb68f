"""Outline obstacles in the batched world on the GPU: scans and steps against the float64 oracle (oracle/world.py),
the old entry point against nb_world_set_scenes_ex, closed-loop runs of PlannerBatch in seeded non_obs / dyna_non_obs scenes,
determinism and the absence of host synchronisation."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from gpu_helpers import record
from helpers import CONFIGS, weights_path
from neupan_b200 import PlannerBatch, WorldBatch, _lib, rollout
from neupan_b200.robot import robot as Robot
from neupan_b200.world import dyna_non_obs, non_obs, pack_scenes, pack_scenes_ex, random_outline
from test_gpu_world import EXAMPLE_LIDAR, LIDAR, _mixed_scenes, _oracle_cfg, _polygon, _ulps
from oracle.world import OracleWorld

pytestmark = pytest.mark.gpu


def _outline(rng):
    return random_outline(rng, rng.uniform(0.3, 1.5), rng.uniform(0.0, 1.0), rng.uniform(0.0, 1.0), int(rng.integers(3, 17)))


def _outline_scenes(B, seed, speed=0.5):
    """Random circles, convex polygons and outlines (3..16 vertices) around the robot; environment 0 at the edge limit (128
    outlines of 16 vertices = 2048 edges)."""
    scenes = []
    for b in range(B):
        rng = np.random.default_rng([seed, b])
        n = 128 if b == 0 else int(rng.integers(1, 30))
        obs = []
        for _ in range(n):
            c, v = tuple(rng.uniform(-12, 12, 2)), tuple(rng.uniform(-speed, speed, 2))
            u = rng.uniform()
            if b == 0:
                obs.append(dict(center=c, outline=random_outline(rng, rng.uniform(0.3, 1.5), 1.0, 0.5, 16), velocity=v))
            elif u < 0.5:
                obs.append(dict(center=c, outline=_outline(rng), velocity=v))
            elif u < 0.75:
                obs.append(dict(center=c, radius=rng.uniform(0.2, 1.5), velocity=v))
            else:
                obs.append(dict(center=c, vertices=_polygon(rng), velocity=v))
        scenes.append(dict(obstacles=obs, bounds=(-12.0, -12.0, 12.0, 12.0), start=(rng.uniform(-3, 3), rng.uniform(-3, 3), rng.uniform(-np.pi, np.pi)),
                           goal=(rng.uniform(-5, 5), rng.uniform(-5, 5)), goal_threshold=0.5))
    return scenes


@pytest.mark.parametrize("R", [37, 1080])
def test_scan_with_outlines_matches_the_oracle(R):
    B = 128
    rb = Robot(10, 0.1, kinematics="diff", length=1.6, width=2.0)
    lidar = dict(LIDAR, number=R, scan_offset=(0.2, -0.1, 0.05))
    scenes = _outline_scenes(B, 300 + R)
    packed = pack_scenes_ex(scenes)
    assert packed[0][1] == 128 and packed[2][128] == 2048  # environment 0 sits at the edge limit
    w = WorldBatch(B, rb, lidar, 0.1)
    w.set_scenes(scenes)
    ranges, vel, _, hit = w.scan(hit=True)
    ranges, vel, hit = ranges.cpu().numpy(), vel.cpu().numpy(), hit.cpu().numpy()
    r64, v64, h64, tie, tan_ = OracleWorld(_oracle_cfg(rb, lidar), packed).scan()
    excused = tie | tan_
    same = hit == h64
    ulps = _ulps(ranges, r64.astype(np.float32))
    kinds = packed[5]
    on_outline = np.array([[h >= 0 and kinds[packed[0][b] + h] == 1 for h in h64[b]] for b in range(B)])
    record(f"world_outline_scan_R{R}", beams=B * R, hits=int((h64 >= 0).sum()), outline_hits=int(on_outline.sum()), excused=int(excused.sum()),
           hit_mismatch_excused=int(((hit != h64) & excused).sum()), max_ulps=int(ulps[same].max()), ulp1=int((ulps[same] == 1).sum()))
    assert not ((hit != h64) & ~excused).any(), np.argwhere((hit != h64) & ~excused)[:5]
    assert not (same & (ulps > 1)).any()
    assert not (same[:, None, :].repeat(2, 1) & (vel != v64.astype(np.float32))).any()
    assert on_outline.mean() > 0.2 and on_outline[0].mean() > 0.2
    w.close()


@pytest.mark.parametrize("kin", ["diff", "acker", "omni"])
def test_steps_with_outlines_match_the_oracle(kin):
    B, steps = 64, 50
    kw = dict(kinematics=kin, length=4.6, width=1.6, wheelbase=3) if kin == "acker" else dict(kinematics=kin, length=1.6, width=2.0)
    if kin == "omni":
        kw = dict(kinematics=kin, vertices=[[-0.8, -1.0], [-1.8, 1.0], [1.8, 1.0], [0.8, -1.0]])
    rb = Robot(10, 0.1, **kw)
    lidar = dict(LIDAR, number=16)
    scenes = _outline_scenes(B + 1, 17, speed=3.0)[1:]
    w = WorldBatch(B, rb, lidar, 0.1)
    w.set_scenes(scenes)
    o = OracleWorld(_oracle_cfg(rb, lidar), pack_scenes_ex(scenes))
    rng = np.random.default_rng(6)
    worst, ulp1, ncol, nclear = 0.0, 0, 0, 0
    for k in range(steps):
        act = np.column_stack([rng.uniform(-1, 2, B), rng.uniform(-0.5, 0.5, B)]).astype(np.float32)
        col, arr, clear = w.step(torch.from_numpy(act).cuda())
        c_o, a_o, clear_o = o.step(act)
        assert np.array_equal(col.cpu().numpy(), c_o) and np.array_equal(arr.cpu().numpy(), a_o)
        assert np.array_equal(w.obstacles().cpu().numpy(), o.obs)
        u = _ulps(clear.cpu().numpy(), clear_o.astype(np.float32))
        assert (u <= 1).all(), (k, np.flatnonzero(u > 1))
        ulp1 += int((u == 1).sum())
        nclear += int((clear_o > 0).sum())
        worst = max(worst, float(np.abs(w.states.cpu().numpy() - o.states).max()))
        ncol = int(c_o.sum())
    record(f"world_outline_step_{kin}", steps=steps, envs=B, max_state_err=worst, clearance_ulp1=ulp1, collided_at_end=ncol,
           positive_clearances=nclear)
    assert worst <= 1e-12
    assert 0 < ncol < B
    w.close()


def _set_scenes_old(w, scenes):
    """WorldBatch.set_scenes through the entry point without kinds (nb_world_set_scenes)."""
    packed = pack_scenes(scenes)
    with torch.cuda.device(w.device):
        _lib.check(_lib.load().nb_world_set_scenes(w._handle, w.B, *[C.c_void_p(a.ctypes.data) for a in packed]))
    w.O = int(packed[0][-1])


def test_old_and_ex_entry_points_agree_bit_for_bit_on_convex_scenes():
    B = 64
    rb = Robot(10, 0.1, kinematics="diff", length=1.6, width=2.0)
    lidar = dict(LIDAR, number=360, scan_offset=(0.2, -0.1, 0.05))
    scenes = _mixed_scenes(B, 41, speed=3.0)
    old, ex = WorldBatch(B, rb, lidar, 0.1), WorldBatch(B, rb, lidar, 0.1)
    _set_scenes_old(old, scenes)
    ex.set_scenes(scenes)
    rng = np.random.default_rng(8)
    for _ in range(20):
        a, b = old.scan(hit=True), ex.scan(hit=True)
        assert all(torch.equal(x, y) for x, y in zip(a, b) if torch.is_tensor(x))
        act = torch.from_numpy(np.column_stack([rng.uniform(-1, 2, B), rng.uniform(-0.5, 0.5, B)]).astype(np.float32)).cuda()
        a, b = old.step(act), ex.step(act)
        assert all(torch.equal(x, y) for x, y in zip(a, b))
        assert torch.equal(old.states, ex.states) and torch.equal(old.obstacles(), ex.obstacles())
    assert all(torch.equal(x, y) for x, y in zip(old.flags(), ex.flags()))
    old.close(); ex.close()


def _planner(cfg_id, B, lidar):
    cfg = CONFIGS[cfg_id]
    return PlannerBatch(B, cfg.T, cfg.dt, 4.0, robot_kwargs=cfg.robot_kwargs, adjust_kwargs=dict(cfg.adjust),
                        pan_kwargs=dict(iter_num=cfg.K, dune_max_num=lidar["number"], nrmp_max_num=cfg.M, dune_checkpoint=weights_path(cfg.model),
                                        iter_threshold=0.0, max_points=lidar["number"]))


def _closed_loop(cfg_id, scenes, steps, blind=False):
    B = len(scenes)
    pl = _planner(cfg_id, B, EXAMPLE_LIDAR)
    pl.set_initial_paths([sc["path"] for sc in scenes])
    w = WorldBatch(B, pl.robot, EXAMPLE_LIDAR, pl.dt)
    w.set_scenes(scenes)
    out = rollout(pl, w, steps, blind=blind)
    out = {k: v.cpu().numpy() for k, v in out.items()}
    out["states"] = w.states.cpu().numpy()
    out["obstacles"] = w.obstacles().cpu().numpy()
    pl.close(); w.close()
    return out


# (scene builder, config after the example it follows, steps, thresholds: blind collisions at least, collisions with scans at
# most, arrivals with scans at least).  Observed on an H100 (of 128): dyna_non_obs 117 blind, 5 with scans, 116 arrived;
# non_obs 128 blind, 2 with scans, 61 arrived (the acker robot's other runs neither collide nor reach the goal in 200 steps).
CLOSED_LOOP = {
    "dyna_non_obs": (dyna_non_obs, "C4", 200, 100, 12, 100),
    "non_obs": (non_obs, "C3", 200, 120, 8, 50),
}


@pytest.mark.parametrize("scene", list(CLOSED_LOOP))
def test_closed_loop_robots_avoid_outline_obstacles_they_see(scene):
    builder, cfg_id, steps, min_blind, max_seen, min_arrived = CLOSED_LOOP[scene]
    scenes = builder(128, seed=2024)
    seen = _closed_loop(cfg_id, scenes, steps)
    blind = _closed_loop(cfg_id, scenes, steps, blind=True)
    n_seen, n_blind = int(seen["collided"].sum()), int(blind["collided"].sum())
    arrived = seen["steps_to_arrive"][seen["arrived"]]
    record(f"world_closed_loop_{scene}", envs=128, steps=steps, config=cfg_id, collided_with_scans=n_seen, collided_blind=n_blind,
           arrived_with_scans=int(seen["arrived"].sum()), arrived_blind=int(blind["arrived"].sum()),
           max_steps_to_arrive=int(arrived.max()) if len(arrived) else -1, min_clearance_median=float(np.median(seen["min_clearance"])))
    assert n_blind >= min_blind and n_seen <= max_seen and int(seen["arrived"].sum()) >= min_arrived


def test_rollouts_with_outlines_are_deterministic():
    scenes = dyna_non_obs(32, seed=5)
    a, b = _closed_loop("C4", scenes, 30), _closed_loop("C4", scenes, 30)
    for k in ("states", "obstacles", "collided", "arrived", "steps_to_arrive", "min_clearance"):
        assert np.array_equal(a[k], b[k]), k


class _StillPlanner:
    def __init__(self, B):
        self.zero = torch.zeros(B, 2, device="cuda")

    def forward(self, states, ranges, scan, scan_offset=None, scan_velocity=None):
        return self.zero, {}


def test_world_with_outlines_does_not_synchronise_the_host():
    B = 64
    rb = Robot(10, 0.1, kinematics="diff", length=1.6, width=2.0)
    w = WorldBatch(B, rb, EXAMPLE_LIDAR, 0.1)
    w.set_scenes(dyna_non_obs(B, seed=1))
    action = torch.zeros(B, 2, device="cuda")
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            ranges, vel, scan = w.scan()
            col, arr, clear = w.step(action)
            _ = w.states
        out = rollout(_StillPlanner(B), w, 5)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert out["min_clearance"].shape == (B,)
    w.close()
