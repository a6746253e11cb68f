"""Several robots per environment in the batched world on the GPU: a fleet of one against the single-robot world (bitwise, and the
same launches), teacher-forced parity of the scan, the fleet step and the reactive obstacles against tests/world_fleet_oracle.py,
edge cases, and closed-loop circle_swap runs of 1024 planners with and without point velocities."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from gpu_helpers import record
from helpers import CONFIGS, weights_path
from neupan_b200 import PlannerBatch, WorldBatch, _lib, rollout
from neupan_b200.robot import robot as Robot
from neupan_b200.world import circle_swap, pack_behaviors, pack_fleet, pack_scenes_ex, random_outline, scene_paths
from oracle import world as ow
from test_gpu_world import EXAMPLE_LIDAR, LIDAR, _mixed_scenes, _oracle_cfg, _polygon, _ulps
from test_gpu_world_outline import _StillPlanner
from test_gpu_world_rvo import ROBOT_KW, _behavior, _rvo_scenes
from world_fleet_oracle import OracleWorld, clearance_robot_pairs

pytestmark = pytest.mark.gpu


def _set_fleet(w, K, rows):
    rows = np.ascontiguousarray(np.asarray(rows, np.float64).reshape(-1, 6))
    with torch.cuda.device(w.device):
        _lib.check(_lib.load().nb_world_set_fleet(w._handle, w.B, K, C.c_void_p(rows.ctypes.data)))
    w.K, w.N = K, w.B * K


# ---- 1. a fleet of one is the single-robot world ---------------------------------------------------------------------------

@pytest.mark.parametrize("reactive", [False, True])
def test_fleet_of_one_is_the_single_robot_world(reactive):
    B = 64
    rb = Robot(10, 0.1, **ROBOT_KW["diff"])
    lidar = dict(LIDAR, number=360, scan_offset=(0.2, -0.1, 0.05))
    scenes = _rvo_scenes(B, 23) if reactive else _mixed_scenes(B + 2, 9)[2:]
    plain, fleet = WorldBatch(B, rb, lidar, 0.1), WorldBatch(B, rb, lidar, 0.1)
    plain.set_scenes(scenes, seed=5)
    fleet.set_scenes(scenes, seed=5)
    _set_fleet(fleet, 1, pack_scenes_ex(scenes)[4][:, 4:10])
    lib = _lib.load()
    rng = np.random.default_rng(6)
    per_call = 3 if reactive else 2
    for _ in range(50):
        act = torch.from_numpy(np.column_stack([rng.uniform(-1, 2, B), rng.uniform(-0.5, 0.5, B)]).astype(np.float32)).cuda()
        n0 = lib.nb_launch_count()
        a = plain.scan(hit=True) + plain.step(act)
        n1 = lib.nb_launch_count()
        b = fleet.scan(hit=True) + fleet.step(act)
        n2 = lib.nb_launch_count()
        assert n1 - n0 == n2 - n1 == per_call  # the world without a fleet launches what it did before: scan, (rvo,) step
        assert all(torch.equal(x, y) for x, y in zip(a, b) if torch.is_tensor(x))
        assert torch.equal(plain.states, fleet.states) and torch.equal(plain.obstacles(), fleet.obstacles())
    assert all(torch.equal(x, y) for x, y in zip(plain.flags(), fleet.flags()))
    if reactive:
        assert all(torch.equal(x, y) for x, y in zip(plain.goals(), fleet.goals()))
    c, _ = plain.flags()
    record(f"world_fleet_of_one_reactive{int(reactive)}", envs=B, steps=50, collided=int(c.sum()))
    plain.close(); fleet.close()


# ---- 2. teacher-forced parity ----------------------------------------------------------------------------------------------

def _fleet_scenes(B, K, seed, rb):
    """Mixed obstacles (circles, convex polygons, outlines; about half reactive) in [-12, 12]^2 and K robots placed at random in
    [-8, 8]^2 with start bodies at least 0.3 m apart."""
    rv = np.asarray(rb.vertices, np.float64).T
    scenes = []
    for b in range(B):
        rng = np.random.default_rng([seed, K, b])
        obs = []
        for _ in range(int(rng.integers(0, 7))):
            ob = dict(center=tuple(rng.uniform(-11.5, 11.5, 2)), velocity=tuple(rng.uniform(-0.5, 0.5, 2)))
            u = rng.uniform()
            if u < 0.4:
                ob["radius"] = rng.uniform(0.2, 1.0)
            elif u < 0.7:
                ob["vertices"] = _polygon(rng) * 0.7
            else:
                ob["outline"] = random_outline(rng, rng.uniform(0.3, 1.0), rng.uniform(0.0, 1.0), rng.uniform(0.0, 1.0), int(rng.integers(3, 17)))
            if rng.uniform() < 0.5:
                ob["behavior"] = _behavior(rng, rng.uniform(2.0, 8.0))
            obs.append(ob)
        robots, bodies = [], []
        while len(robots) < K:
            s = (rng.uniform(-8, 8), rng.uniform(-8, 8), rng.uniform(-np.pi, np.pi))
            body = np.asarray(ow.robot_polygon(s, rv))
            if bodies and clearance_robot_pairs(np.repeat(body[None], len(bodies), 0), np.asarray(bodies)).min() < 0.3:
                continue
            bodies.append(body)
            robots.append(dict(start=s, goal=tuple(rng.uniform(-8, 8, 2)), goal_threshold=rng.uniform(0.3, 1.0), path=None))
        scenes.append(dict(obstacles=obs, bounds=(-12.0, -12.0, 12.0, 12.0), robots=robots))
    return scenes


def _actions(rng, kin, states, K):
    """Random actions; about a third of the robots steer towards the nearest other robot of their environment."""
    N = len(states)
    v = rng.uniform(-1.0, 2.5, N)
    w = rng.uniform(-0.5, 0.5, N)
    xy = states[:, :2].reshape(-1, K, 2)
    d = np.linalg.norm(xy[:, :, None] - xy[:, None], axis=3) + np.eye(K) * 1e9
    tgt = xy[np.arange(len(xy))[:, None], d.argmin(2)].reshape(N, 2)
    chase = rng.uniform(size=N) < 0.35
    dx, dy = tgt[:, 0] - states[:, 0], tgt[:, 1] - states[:, 1]
    err = np.angle(np.exp(1j * (np.arctan2(dy, dx) - states[:, 2])))
    if kin == "omni":
        nrm = np.maximum(np.hypot(dx, dy), 1e-9)
        act = np.column_stack([np.where(chase, 2.5 * dx / nrm, v), np.where(chase, 2.5 * dy / nrm, w * 4)])
    else:
        act = np.column_stack([np.where(chase, 2.5, v), np.where(chase, np.clip(2.0 * err, -0.5, 0.5), w)])
    return act.astype(np.float32)


def _device(w):
    g, d = w.goals()
    c, a = w.flags()
    return dict(obs=w.obstacles().cpu().numpy(), states=w.states.cpu().numpy(), collided=c.cpu().numpy(), arrived=a.cpu().numpy(),
                goal=g.cpu().numpy(), draws=d.cpu().numpy())


@pytest.mark.parametrize("K", [2, 5, 16])
@pytest.mark.parametrize("kin", ["diff", "acker", "omni"])
def test_teacher_forced_fleet_matches_the_oracle(kin, K):
    """50 steps of B = 128 mixed scenes: before every step the oracle takes the device's state; then scans (hit, ranges, velocity),
    the reactive obstacles' choices, the robots' states, flags and clearances must agree.  Excuses: a beam within 1e-9 m of two
    crossings or tangent to a circle (the scan tests' excuse), a reactive obstacle whose decision involved a robot with a margin below
    1e-12 (the reactive tests' excuse); the robots' velocities and bodies use CUDA's sincos there and libm here."""
    B, steps = 128, 50
    rb = Robot(10, 0.1, **ROBOT_KW[kin])
    lidar = dict(LIDAR, number=16, scan_offset=(0.1, 0.05, 0.1))
    scenes = _fleet_scenes(B, K, 71, rb)
    packed, beh, fleet = pack_scenes_ex(scenes), pack_behaviors(scenes), pack_fleet(scenes)
    w = WorldBatch(B, rb, lidar, 0.1)
    w.set_scenes(scenes, seed=13)
    assert (w.K, w.N) == (K, B * K)
    o = OracleWorld(_oracle_cfg(rb, lidar), packed, fleet, K, beh, seed=13)
    rng = np.random.default_rng(17)
    robot_hits = robot_collisions = excused_beams = excused_obs = worst_state = ulp1 = 0
    wrong = []
    for k in range(steps):
        s = _device(w)
        o.obs[:], o.states[:], o.collided[:], o.arrived[:], o.goal[:], o.draws[:] = (s["obs"], s["states"], s["collided"], s["arrived"],
                                                                                     s["goal"], s["draws"])
        ranges, vel, _, hit = (t.cpu().numpy() if torch.is_tensor(t) else t for t in w.scan(hit=True))
        r64, v64, h64, tie, tan_ = o.scan()
        exc = tie | tan_
        same = hit == h64
        assert not (~same & ~exc).any(), (k, np.argwhere(~same & ~exc)[:5])
        excused_beams += int((~same).sum())
        assert (_ulps(ranges, r64.astype(np.float32))[same] <= 1).all(), k
        assert np.array_equal(vel[np.repeat(same[:, None], 2, 1)], v64.astype(np.float32)[np.repeat(same[:, None], 2, 1)]), k
        nobs = np.repeat(np.diff(o.obs_begin), K)[:, None]
        robot_hits += int((h64 >= nobs).sum())
        act = _actions(rng, kin, s["states"], K)
        margins = o.rvo(act)
        _, _, clear_o = o.step(act, rvo=False)
        col, arr, clear = (t.cpu().numpy() for t in w.step(torch.from_numpy(act).cuda()))
        d = _device(w)
        bad_env = set()
        for b in range(B):
            sl = slice(o.obs_begin[b], o.obs_begin[b + 1])
            bad = ~(np.all(d["obs"][sl] == o.obs[sl], 1) & np.all(d["goal"][sl] == o.goal[sl], 1) & (d["draws"][sl] == o.draws[sl]))
            for q in np.flatnonzero(bad) + sl.start:
                if margins[q] < 1e-12:
                    excused_obs += 1
                    bad_env.add(b)
                else:
                    wrong.append(("obstacle", k, b, int(q)))
        ok = np.ones(B * K, bool)
        for b in bad_env:  # an excused obstacle moved elsewhere: that environment's robots are not compared this step
            ok[b * K:(b + 1) * K] = False
        worst_state = max(worst_state, float(np.abs(d["states"] - o.states)[ok].max()))
        assert np.array_equal(col[ok], o.collided[ok]) and np.array_equal(arr[ok], o.arrived[ok]), k
        assert np.array_equal(d["collided"], col) and np.array_equal(d["arrived"], arr)
        u = _ulps(clear, clear_o.astype(np.float32))[ok]
        assert (u <= 1).all(), (k, np.flatnonzero(u > 1)[:5])
        ulp1 += int((u == 1).sum())
        robot_collisions += int(((o.robot_clear <= 0.0) & (s["collided"] == 0)).sum())
    record(f"world_fleet_teacher_forced_{kin}_K{K}", envs=B, robots=B * K, steps=steps, beams=steps * B * K * 16, robot_hits=robot_hits,
           robot_robot_collisions=robot_collisions, collided_at_end=int(o.collided.sum()), excused_beams=excused_beams,
           excused_obstacles=excused_obs, max_state_err=worst_state, clearance_ulp1=ulp1, mismatches=len(wrong))
    assert not wrong, wrong[:3]
    assert worst_state <= 1e-12
    assert robot_hits > 0 and robot_collisions > 0  # OBSERVED: both are reported above
    w.close()


# ---- 3. edge cases -----------------------------------------------------------------------------------------------------------

def _scene(robots, obstacles=(), ext=30.0):
    return dict(obstacles=list(obstacles), bounds=(-ext, -ext, ext, ext),
                robots=[dict(start=s, goal=(50.0, 50.0), goal_threshold=0.1, path=None) for s in robots])


def test_a_robot_never_sees_itself():
    B, K = 4, 3
    rb = Robot(10, 0.1, **ROBOT_KW["diff"])
    for off in ((0.0, 0.0, 0.0), (0.5, 0.3, 0.7)):  # a sensor inside its own body
        lidar = dict(LIDAR, number=720, range_max=5.0, scan_offset=off)
        scenes = [_scene([(-20.0, 0.0, 0.1 * b), (0.0, 20.0, 1.0), (20.0, -20.0, -2.0)]) for b in range(B)]
        w = WorldBatch(B, rb, lidar, 0.1)
        w.set_scenes(scenes)
        ranges, vel, _, hit = w.scan(hit=True)
        assert (hit == -1).all() and (ranges == 5.0).all() and not vel.any()
        w.close()


def test_robot_hits_report_the_index_and_velocity_and_collided_robots_stay():
    """Robots 0 and 1 drive at each other head-on along y = 0; robot 2 drives into a wall; the environment has two obstacles (a far
    circle and the wall), so robot 1 is hit index 2 + 1.  Checked against the oracle at every step, and directly: robot 1's index and
    its velocity (0 before the first step, the action's after it, 0 once collided); the collision of robots 0 and 1 in the same step;
    collided robots frozen and still seen."""
    rb = Robot(10, 0.1, **ROBOT_KW["diff"])
    lidar = dict(LIDAR, number=9, range_max=20.0)  # beam 4 points along the heading
    wall = dict(center=(0.0, -12.0), vertices=[[-8.0, -0.5], [8.0, -0.5], [8.0, 0.5], [-8.0, 0.5]])
    far = dict(center=(25.0, 25.0), radius=0.5)
    sc = dict(obstacles=[far, wall], bounds=(-30.0, -30.0, 30.0, 30.0),
              robots=[dict(start=s, goal=(50.0, 50.0), goal_threshold=0.1, path=None) for s in ((0.0, 0.0, 0.0), (6.0, 0.0, math.pi), (0.0, -8.0, -math.pi / 2))])
    w = WorldBatch(1, rb, lidar, 0.1)
    w.set_scenes([sc])
    o = OracleWorld(_oracle_cfg(rb, lidar), pack_scenes_ex([sc]), pack_fleet([sc]), 3)
    act = np.array([[1.0, 0.0], [1.5, 0.0], [2.0, 0.0]], np.float32)
    collided_at, seen_after = None, 0
    for k in range(40):
        ranges, vel, hit = (t.cpu().numpy() for t in w.scan(hit=True) if torch.is_tensor(t))
        r64, v64, h64, _, _ = o.scan()
        assert np.array_equal(hit, h64) and (_ulps(ranges, r64.astype(np.float32)) <= 1).all() and np.array_equal(vel, v64.astype(np.float32))
        beams = np.flatnonzero(hit[0] == 3)  # robot 1 = index O_b + 1 = 3 (two obstacles)
        if k == 0:
            assert len(beams) and not vel[0][:, beams].any()  # no step yet: velocity 0
        if k == 1:
            assert len(beams) and (vel[0][0, beams] == -1.5).all()  # robot 1's action (1.5, 0) at heading pi
        col, arr, clear = (t.cpu().numpy() for t in w.step(torch.from_numpy(act).cuda()))
        c_o, _, clear_o = o.step(act)
        assert np.array_equal(col, c_o) and (_ulps(clear, clear_o.astype(np.float32)) <= 1).all()
        if collided_at is None and col[:2].any():
            collided_at = k
            assert col[0] == col[1] == 1  # head-on: both in the same step
        if collided_at is not None and k > collided_at:
            seen_after += int((hit[0] == 3).any())
            assert not vel[0][:, hit[0] == 3].any()  # a collided robot has velocity 0
    assert collided_at is not None and seen_after > 0
    assert col[2] == 1  # robot 2 reached the wall
    frozen = w.states.cpu().numpy()
    w.step(torch.from_numpy(act).cuda())
    assert np.array_equal(w.states.cpu().numpy(), frozen)  # every robot collided: frozen
    record("world_fleet_head_on", collided_at_step=collided_at + 1, seen_after_collision=seen_after)
    w.close()


def test_robot_velocity_in_the_scan_is_the_last_action():
    rb = Robot(10, 0.1, **ROBOT_KW["omni"])
    lidar = dict(LIDAR, number=4, range_max=20.0)  # beams at -pi, -pi/3, pi/3, pi
    sc = _scene([(0.0, 0.0, 0.0), (-8.0, 0.0, 0.0)])
    w = WorldBatch(1, rb, lidar, 0.1)
    w.set_scenes([sc])
    _, vel, _, hit = w.scan(hit=True)
    assert hit[0, 0] == 1 and hit[0, 3] == 1 and not vel.any()  # robot 1 behind robot 0, index 0 + 1
    w.step(torch.tensor([[0.0, 0.0], [0.25, -0.5]], device="cuda"))
    _, vel, _, hit = w.scan(hit=True)
    assert hit[0, 0] == 1 and vel[0, :, 0].tolist() == [0.25, -0.5]
    w.close()


def test_an_obstacle_wins_a_tie_with_a_robot_and_a_sensor_inside_a_robot_sees_the_exit():
    rb = Robot(10, 0.1, kinematics="diff", length=1.6, width=2.0)
    rv = np.asarray(rb.vertices, np.float64).T
    # obstacle 0: exactly robot 1's body at (5, 0, 0) (cos 0 = 1, sin 0 = 0: the same world vertices bit for bit)
    twin = dict(center=(5.0, 0.0), vertices=rv)
    lidar = dict(LIDAR, number=1, angle_min=0.0, angle_max=0.0, range_max=20.0)
    w = WorldBatch(1, rb, lidar, 0.1)
    w.set_scenes([_scene([(0.0, 0.0, 0.0), (5.0, 0.0, 0.0)], [twin])])
    ranges, _, _, hit = w.scan(hit=True)
    assert hit[:, 0].tolist() == [0, 0] and ranges[0, 0].item() == np.float32(5.0 - 0.8 - 0.0)  # robot 0 sees the obstacle, not robot 1
    w.close()
    inside = dict(LIDAR, number=2, angle_min=0.0, angle_max=math.pi, range_max=20.0, scan_offset=(2.5, 0.0, 0.0))
    w = WorldBatch(1, rb, inside, 0.1)
    sc = _scene([(0.0, 0.0, 0.0), (2.6, 0.0, 0.0)])
    w.set_scenes([sc])
    ranges, _, _, hit = w.scan(hit=True)
    o = OracleWorld(_oracle_cfg(rb, inside), pack_scenes_ex([sc]), pack_fleet([sc]), 2)
    r64, _, h64, _, _ = o.scan()
    assert hit[0].tolist() == [1, 1] == h64[0].tolist()  # the sensor sits inside robot 1: both beams see its exit crossings
    assert abs(ranges[0, 0].item() - 0.9) < 1e-6 and abs(ranges[0, 1].item() - 0.7) < 1e-6
    assert np.array_equal(ranges.cpu().numpy(), r64.astype(np.float32))
    w.close()


def test_fleet_handles_of_different_sizes_coexist():
    """The scan's dynamic shared memory includes the robot edges; each handle sets its own size before every launch."""
    rb = Robot(10, 0.1, **ROBOT_KW["diff"])
    big = WorldBatch(8, rb, EXAMPLE_LIDAR, 0.1)
    big.set_scenes(_fleet_scenes(8, 16, 3, rb))
    small = WorldBatch(8, rb, EXAMPLE_LIDAR, 0.1)
    small.set_scenes(_fleet_scenes(8, 2, 4, rb))
    plain = WorldBatch(8, rb, EXAMPLE_LIDAR, 0.1)
    plain.set_scenes(_mixed_scenes(8, 5))
    first = [[t.cpu() for t in w.scan(hit=True) if torch.is_tensor(t)] for w in (big, small, plain)]
    for w, ref in zip((big, small, plain), first):
        assert all(torch.equal(t.cpu(), r) for t, r in zip((t for t in w.scan(hit=True) if torch.is_tensor(t)), ref))
    assert first[0][0].shape == (8 * 16, 100) and first[1][0].shape == (16, 100) and first[2][0].shape == (8, 100)
    with pytest.raises(ValueError, match="count = 8 but the world has 8 environments x 16 robots"):
        _lib.check(_lib.load().nb_world_scan(big._handle, 8, C.c_void_p(first[0][0].data_ptr()), None, None, None))
    for w in (big, small, plain):
        w.close()


# ---- 4. closed loop ----------------------------------------------------------------------------------------------------------

def _planner(N):
    cfg = CONFIGS["C4"]
    return PlannerBatch(N, cfg.T, cfg.dt, 4.0, robot_kwargs=cfg.robot_kwargs, adjust_kwargs=dict(cfg.adjust),
                        pan_kwargs=dict(iter_num=cfg.K, dune_max_num=EXAMPLE_LIDAR["number"], nrmp_max_num=cfg.M,
                                        dune_checkpoint=weights_path(cfg.model), iter_threshold=0.0, max_points=EXAMPLE_LIDAR["number"]))


def _swap_loop(scenes, steps, **kw):
    B, K = len(scenes), len(scenes[0]["robots"])
    pl = _planner(B * K)
    pl.set_initial_paths(scene_paths(scenes))
    w = WorldBatch(B, pl.robot, EXAMPLE_LIDAR, pl.dt)
    w.set_scenes(scenes)
    out = rollout(pl, w, steps, **kw)
    out = {k: v.cpu().numpy() for k, v in out.items()}
    out["states"] = w.states.cpu().numpy()
    # a collided robot is frozen where it collided; it hit a robot if it overlaps one there, otherwise an obstacle
    rv = np.asarray(pl.robot.vertices, np.float64).T
    bodies = np.array([ow.robot_polygon(s, rv) for s in out["states"]]).reshape(B, K, -1, 2)
    ii, jj = np.nonzero(~np.eye(K, dtype=bool))
    rr = np.stack([clearance_robot_pairs(bodies[b, ii], bodies[b, jj]).reshape(K, K - 1).min(1) for b in range(B)]).reshape(-1)
    out["robot_robot"] = out["collided"] & (rr <= 0.0)
    pl.close(); w.close()
    return out


# Observed on one H100 (1024 robots, 120 steps): with point velocities 335 robots collide (all robot-robot) and 350 arrive, the
# median after 75 steps; without them and blind all 1024 collide and none arrives.  The thresholds sit just below.
SWAP_STEPS = 120


def test_closed_loop_circle_swap():
    scenes = circle_swap(128, robots=8, seed=2024)
    legs = {"velocities": _swap_loop(scenes, SWAP_STEPS), "no_velocities": _swap_loop(scenes, SWAP_STEPS, velocities=False),
            "blind": _swap_loop(scenes, SWAP_STEPS, blind=True)}
    again = _swap_loop(scenes, SWAP_STEPS)
    for k in ("states", "collided", "arrived", "steps_to_arrive", "min_clearance"):
        assert np.array_equal(legs["velocities"][k], again[k]), k
    summary = {}
    for name, out in legs.items():
        arrived = out["steps_to_arrive"][out["arrived"]]
        summary[name] = dict(collided_robot_robot=int(out["robot_robot"].sum()), collided_robot_obstacle=int((out["collided"] & ~out["robot_robot"]).sum()),
                             arrived=int(out["arrived"].sum()), median_steps_to_arrive=float(np.median(arrived)) if len(arrived) else -1.0,
                             max_steps_to_arrive=int(arrived.max()) if len(arrived) else -1,
                             min_clearance_median=float(np.median(out["min_clearance"])))
    record("world_fleet_closed_loop_circle_swap", envs=128, robots=1024, steps=SWAP_STEPS, config="C4", **summary)
    assert summary["velocities"]["arrived"] >= 330 and summary["velocities"]["collided_robot_robot"] <= 360
    assert summary["no_velocities"]["collided_robot_robot"] >= 1000 and summary["blind"]["collided_robot_robot"] >= 1000


def test_fleet_rollout_does_not_synchronise_the_host():
    B, K = 32, 8
    rb = Robot(10, 0.1, **ROBOT_KW["diff"])
    w = WorldBatch(B, rb, EXAMPLE_LIDAR, 0.1)
    w.set_scenes(circle_swap(B, robots=K, seed=1))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = rollout(_StillPlanner(B * K), w, 5)
        out = rollout(_StillPlanner(B * K), w, 5, velocities=False)
        out = rollout(_StillPlanner(B * K), w, 5, blind=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert out["min_clearance"].shape == (B * K,)
    w.close()
