"""The batched world on the GPU: scans and steps against the float64 oracle (oracle/world.py), the scan -> points chain, closed-loop
runs of PlannerBatch in seeded dyna_obs / corridor scenes, determinism and the absence of host synchronisation."""
import math

import numpy as np
import pytest
import torch

from gpu_helpers import record
from helpers import CONFIGS, weights_path
from neupan_b200 import PlannerBatch, WorldBatch, rollout, scan_to_points
from neupan_b200.robot import robot as Robot
from neupan_b200.world import corridor, dyna_obs, pack_scenes
from oracle import world as ow

pytestmark = pytest.mark.gpu

LIDAR = dict(angle_min=-math.pi, angle_max=math.pi, range_min=0.0, range_max=12.0)
# the lidar2d of example/dyna_obs/diff/env.yaml and example/corridor/diff/env.yaml: 100 beams over pi, range 0..10 m
EXAMPLE_LIDAR = dict(angle_min=-math.pi / 2, angle_max=math.pi / 2, range_min=0.0, range_max=10.0, number=100)


def _oracle_cfg(rb, lidar, dt=0.1):
    return dict(kinematics=rb.kinematics, step_time=dt, wheelbase=rb.L, angle_min=lidar["angle_min"], angle_max=lidar["angle_max"],
                range_max=lidar["range_max"], number=lidar["number"], scan_offset=lidar.get("scan_offset", (0.0, 0.0, 0.0)),
                robot_vertices=np.asarray(rb.vertices, np.float64).T)


def _polygon(rng):
    n = int(rng.integers(3, 9))
    ang = np.sort(rng.uniform(0, 2 * np.pi - 0.01, n)) + np.arange(n) * 1e-3  # strictly increasing on a circle: convex
    rad = rng.uniform(0.3, 1.5)
    return np.stack([rad * np.cos(ang), rad * np.sin(ang)], 1)


def _mixed_scenes(B, seed, speed=0.5):
    """Random circles and convex polygons around the robot; environment 0 at the obstacle limit (256 circles), environment 1 at
    the edge limit (256 octagons = 2048 edges)."""
    octagon = [[math.cos(k * math.pi / 4), math.sin(k * math.pi / 4)] for k in range(8)]
    scenes = []
    for b in range(B):
        rng = np.random.default_rng([seed, b])
        n = 256 if b < 2 else int(rng.integers(1, 30))
        obs = []
        for i in range(n):
            c = tuple(rng.uniform(-12, 12, 2))
            v = tuple(rng.uniform(-speed, speed, 2))
            if b == 0 or (b > 1 and rng.uniform() < 0.5):
                obs.append(dict(center=c, radius=rng.uniform(0.2, 1.5), velocity=v))
            else:
                obs.append(dict(center=c, vertices=np.asarray(octagon) * rng.uniform(0.2, 1.0) if b == 1 else _polygon(rng), velocity=v))
        scenes.append(dict(obstacles=obs, bounds=(-12.0, -12.0, 12.0, 12.0), start=(rng.uniform(-3, 3), rng.uniform(-3, 3), rng.uniform(-np.pi, np.pi)),
                           goal=(rng.uniform(-5, 5), rng.uniform(-5, 5)), goal_threshold=0.5))
    return scenes


def _ulps(a32, b32):
    return np.abs(a32.view(np.int32).astype(np.int64) - b32.view(np.int32).astype(np.int64))


@pytest.mark.parametrize("R", [1, 37, 1080, 4000])
def test_scan_matches_the_oracle(R):
    B = 256
    rb = Robot(10, 0.1, kinematics="diff", length=1.6, width=2.0)
    lidar = dict(LIDAR, number=R, scan_offset=(0.2, -0.1, 0.05))
    scenes = _mixed_scenes(B, 100 + R)
    w = WorldBatch(B, rb, lidar, 0.1)
    w.set_scenes(scenes)
    ranges, vel, _, hit = w.scan(hit=True)
    ranges, vel, hit = ranges.cpu().numpy(), vel.cpu().numpy(), hit.cpu().numpy()
    o = ow.OracleWorld(_oracle_cfg(rb, lidar), pack_scenes(scenes))
    r64, v64, h64, tie, tan_ = o.scan()
    excused = tie | tan_
    bad_hit = (hit != h64) & ~excused
    same = (hit == h64)
    ulps = _ulps(ranges, r64.astype(np.float32))
    bad_range = same & (ulps > 1)
    bad_vel = same[:, None, :].repeat(2, 1) & (vel != v64.astype(np.float32))
    record(f"world_scan_R{R}", beams=B * R, hits=int((h64 >= 0).sum()), excused=int(excused.sum()), hit_mismatch_excused=int(((hit != h64) & excused).sum()),
           max_ulps=int(ulps[same].max()), ulp1=int((ulps[same] == 1).sum()))
    assert not bad_hit.any(), np.argwhere(bad_hit)[:5]
    assert not bad_range.any() and not bad_vel.any()
    assert (h64 >= 0).mean() > 0.3  # the scenes are seen
    w.close()


@pytest.mark.parametrize("kin", ["diff", "acker", "omni"])
def test_steps_match_the_oracle(kin):
    B, steps = 64, 50
    kw = dict(kinematics=kin, length=4.6, width=1.6, wheelbase=3) if kin == "acker" else dict(kinematics=kin, length=1.6, width=2.0)
    if kin == "omni":
        kw = dict(kinematics=kin, vertices=[[-0.8, -1.0], [-1.8, 1.0], [1.8, 1.0], [0.8, -1.0]])
    rb = Robot(10, 0.1, **kw)
    lidar = dict(LIDAR, number=16)
    scenes = _mixed_scenes(B + 2, 7, speed=3.0)[2:]  # fast obstacles: many reflections (the limit environments stay in the scan test)
    w = WorldBatch(B, rb, lidar, 0.1)
    w.set_scenes(scenes)
    o = ow.OracleWorld(_oracle_cfg(rb, lidar), pack_scenes(scenes))
    rng = np.random.default_rng(5)
    worst, ulp1, ncol = 0.0, 0, 0
    for k in range(steps):
        act = np.column_stack([rng.uniform(-1, 2, B), rng.uniform(-0.5, 0.5, B)]).astype(np.float32)
        col, arr, clear = w.step(torch.from_numpy(act).cuda())
        c_o, a_o, clear_o = o.step(act)
        assert np.array_equal(col.cpu().numpy(), c_o) and np.array_equal(arr.cpu().numpy(), a_o)
        assert np.array_equal(w.obstacles().cpu().numpy(), o.obs)
        u = _ulps(clear.cpu().numpy(), clear_o.astype(np.float32))
        assert (u <= 1).all(), (k, np.flatnonzero(u > 1))
        ulp1 += int((u == 1).sum())
        worst = max(worst, float(np.abs(w.states.cpu().numpy() - o.states).max()))
        ncol = int(c_o.sum())
    record(f"world_step_{kin}", steps=steps, envs=B, max_state_err=worst, clearance_ulp1=ulp1, collided_at_end=ncol)
    assert worst <= 1e-12
    w.close()


@pytest.mark.parametrize("velocity_mode", [False, True])
def test_scan_points_lie_on_the_obstacle_boundaries(velocity_mode):
    """scan() -> scan_to_points: scan_to_point applies the sensor offset as s_R p + s_t (neupan.py:216-217), the pose the world casts
    from; scan_to_point_velocity applies its inverse (neupan.py:271-273), so in that mode the chain holds for a sensor at the robot's
    origin only."""
    B = 64
    rb = Robot(10, 0.1, kinematics="diff", length=1.6, width=2.0)
    lidar = dict(LIDAR, number=720, scan_offset=(0.0, 0.0, 0.0) if velocity_mode else (0.3, 0.1, -0.2))
    scenes = _mixed_scenes(B, 21)
    w = WorldBatch(B, rb, lidar, 0.1)
    w.set_scenes(scenes)
    ranges, vel, scan = w.scan()
    pts, pv, cnt = scan_to_points(w.states, ranges, scan, w.scan_offset, velocity=vel if velocity_mode else None)
    pts, cnt = pts.cpu().numpy().astype(np.float64), cnt.cpu().numpy()
    worst, n = 0.0, 0
    for b, sc in enumerate(scenes):
        p = pts[b, :, :cnt[b]].T
        d = np.full(len(p), np.inf)
        for ob in sc["obstacles"]:
            c = np.asarray(ob["center"])
            if "vertices" in ob:
                v = np.asarray(ob["vertices"]) + c
                for k in range(len(v)):
                    a, e = v[k], v[(k + 1) % len(v)] - v[k]
                    t = np.clip(((p - a) @ e) / (e @ e), 0, 1)
                    d = np.minimum(d, np.linalg.norm(p - (a + t[:, None] * e), axis=1))
            else:
                d = np.minimum(d, np.abs(np.linalg.norm(p - c, axis=1) - ob["radius"]))
        worst, n = max(worst, float(d.max()) if len(d) else 0.0), n + len(p)
    record(f"world_scan_chain_velocity_mode{int(velocity_mode)}", points=n, max_boundary_distance=worst)
    assert n > 10000 and worst < 1e-4
    w.close()


def _planner(B, lidar):
    cfg = CONFIGS["C4"]
    return PlannerBatch(B, cfg.T, cfg.dt, 4.0, robot_kwargs=cfg.robot_kwargs, adjust_kwargs=dict(cfg.adjust),
                        pan_kwargs=dict(iter_num=cfg.K, dune_max_num=lidar["number"], nrmp_max_num=cfg.M, dune_checkpoint=weights_path(cfg.model),
                                        iter_threshold=0.0, max_points=lidar["number"]))


def _closed_loop(scenes, steps, blind=False):
    B = len(scenes)
    pl = _planner(B, EXAMPLE_LIDAR)
    pl.set_initial_paths([sc["path"] for sc in scenes])
    w = WorldBatch(B, pl.robot, EXAMPLE_LIDAR, pl.dt)
    w.set_scenes(scenes)
    out = rollout(pl, w, steps, blind=blind)
    out = {k: v.cpu().numpy() for k, v in out.items()}
    out["states"] = w.states.cpu().numpy()
    out["obstacles"] = w.obstacles().cpu().numpy()
    pl.close(); w.close()
    return out


def test_closed_loop_robots_avoid_the_obstacles_they_see():
    scenes = dyna_obs(128, seed=2024)
    steps = 150
    seen = _closed_loop(scenes, steps)
    blind = _closed_loop(scenes, steps, blind=True)
    n_seen, n_blind = int(seen["collided"].sum()), int(blind["collided"].sum())
    record("world_closed_loop_dyna_obs", envs=128, steps=steps, collided_with_scans=n_seen, collided_blind=n_blind,
           arrived_with_scans=int(seen["arrived"].sum()), arrived_blind=int(blind["arrived"].sum()),
           min_clearance_median=float(np.median(seen["min_clearance"])))
    assert n_blind >= 100 and n_seen <= 8  # observed on an H100: 117 blind, 2 with scans (of 128)


def test_closed_loop_corridor_walls_only_every_robot_arrives():
    scenes = corridor(32, seed=7, circles=0)
    budget = 200  # observed on an H100: the last robot arrives after 151 steps
    out = _closed_loop(scenes, budget)
    record("world_closed_loop_corridor", envs=32, budget=budget, arrived=int(out["arrived"].sum()), collided=int(out["collided"].sum()),
           max_steps_to_arrive=int(out["steps_to_arrive"].max()), min_clearance=float(out["min_clearance"].min()))
    assert out["arrived"].all() and not out["collided"].any()


def test_rollouts_are_deterministic():
    scenes = dyna_obs(32, seed=5)
    a, b = _closed_loop(scenes, 30), _closed_loop(scenes, 30)
    for k in ("states", "obstacles", "collided", "arrived", "steps_to_arrive", "min_clearance"):
        assert np.array_equal(a[k], b[k]), k


def test_worlds_with_different_scene_sizes_scan_independently():
    """Each handle stages its own largest environment in shared memory: a later handle with smaller (or empty) scenes must not
    change what an earlier one can launch."""
    B = 16
    rb = Robot(10, 0.1, kinematics="diff", length=1.6, width=2.0)
    empty = [dict(obstacles=[], bounds=(0.0, 0.0, 1.0, 1.0), start=(0.0, 0.0, 0.0), goal=(5.0, 0.0), goal_threshold=0.1)] * B
    worlds, first = [], []
    for scenes in (_mixed_scenes(B, 3), dyna_obs(B, seed=4), corridor(B, seed=5, circles=0), empty):  # largest first
        w = WorldBatch(B, rb, EXAMPLE_LIDAR, 0.1)
        w.set_scenes(scenes)
        worlds.append(w)
        first.append([t.cpu() for t in w.scan(hit=True) if torch.is_tensor(t)])
    for w, ref in zip(worlds, first):
        again = [t.cpu() for t in w.scan(hit=True) if torch.is_tensor(t)]
        assert all(torch.equal(a, r) for a, r in zip(again, ref))
    assert (first[0][2] >= 0).any() and (first[3][2] == -1).all()
    for w in worlds:
        w.close()


class _StillPlanner:
    """A planner that answers zeros on the device: what rollout itself does, without the planner."""

    def __init__(self, B):
        self.zero = torch.zeros(B, 2, device="cuda")

    def forward(self, states, ranges, scan, scan_offset=None, scan_velocity=None):
        return self.zero, {}


def test_world_and_rollout_do_not_synchronise_the_host():
    B = 64
    rb = Robot(10, 0.1, kinematics="diff", length=1.6, width=2.0)
    w = WorldBatch(B, rb, EXAMPLE_LIDAR, 0.1)
    w.set_scenes(dyna_obs(B, seed=1))
    action = torch.zeros(B, 2, device="cuda")
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            ranges, vel, scan = w.scan()
            col, arr, clear = w.step(action)
            _ = w.states
        out = rollout(_StillPlanner(B), w, 5)
        out = rollout(_StillPlanner(B), w, 5, blind=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert out["min_clearance"].shape == (B,)
    w.close()
