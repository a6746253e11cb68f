"""Occupancy maps in the batched world on the GPU: a world whose maps were dropped or that has none in use equals one without
(bitwise, the same launches), teacher-forced parity against the float64 oracle (tests/world_map_oracle.py) for K in {1, 4, 16} and a
mixed fleet with noise, maze and cave maps, edge cases of the grid walk and the windowed clearance, and closed-loop maze and cave
runs of C4's planner."""
import math

import numpy as np
import pytest
import torch

from gpu_helpers import record
from neupan_b200 import WorldBatch, _lib, rollout
from neupan_b200.world import cave, dyna_non_obs, maze, pack_behaviors, pack_fleet, pack_maps, pack_robot_types, pack_scenes_ex
from test_gpu_world import EXAMPLE_LIDAR, LIDAR, _closed_loop, _oracle_cfg, _planner, _ulps
from test_gpu_world_fleet import _device
from test_gpu_world_mixed import _mixed_actions, _mixed_fleet_scenes, _robot, _types_of
from world_map_oracle import MapOracleWorld

pytestmark = pytest.mark.gpu

RESOLUTIONS = (0.05, 0.1, 0.37, 1.0)


def _outputs(w, act):
    a = [t for t in w.scan(hit=True) if torch.is_tensor(t)] + list(w.step(act))
    return a + [w.states, w.obstacles()] + list(w.flags())


# ---- 1. no maps in use: the map-free world -------------------------------------------------------------------------------------

def test_dropped_or_unused_maps_are_the_map_free_world():
    """A handle whose maps set_scenes dropped equals a fresh handle, and one whose every env_map is -1 equals one without maps:
    every output bit for bit over 30 steps, with the same launches."""
    B = 64
    rb = _robot("diff")
    lidar = dict(LIDAR, number=90, scan_offset=(0.2, -0.1, 0.05))
    plain = dyna_non_obs(B, seed=3)
    mazes = maze(B, seed=1)
    fresh, reused, unused = (WorldBatch(B, rb, lidar, 0.1) for _ in range(3))
    fresh.set_scenes(plain, seed=5)
    reused.set_scenes(mazes)
    assert reused.scan(hit=True)[3].max().item() >= 0
    reused.set_scenes(plain, seed=5)  # drops the maps
    unused.set_scenes(plain, seed=5)
    maps, bits, _ = pack_maps(mazes[:1])
    env_map = np.full(B, -1, np.int32)
    with torch.cuda.device(unused.device):
        _lib.check(_lib.load().nb_world_set_maps(unused._handle, 1, maps, bits.ctypes.data, env_map.ctypes.data, 1.0))
    lib = _lib.load()
    rng = np.random.default_rng(2)
    for _ in range(30):
        act = torch.from_numpy(np.column_stack([rng.uniform(-1, 2, B), rng.uniform(-0.5, 0.5, B)]).astype(np.float32)).cuda()
        outs, counts = [], []
        for w in (fresh, reused, unused):
            n0 = lib.nb_launch_count()
            outs.append(_outputs(w, act))
            counts.append(lib.nb_launch_count() - n0)
        assert counts == [2, 2, 2]
        assert all(torch.equal(x, y) for x, y in zip(outs[0], outs[1]))
        assert all(torch.equal(x, y) for x, y in zip(outs[0], outs[2]))
    for w in (fresh, reused, unused):
        w.close()


# ---- 2. teacher-forced parity --------------------------------------------------------------------------------------------------

def _noise_map(rng, res):
    ext = rng.uniform(8.0, 30.0, 2)  # some maps cover only part of the environment
    W, H = (max(1, int(e / res)) for e in ext)
    origin = tuple(rng.uniform(-16.0, 4.0, 2))
    return (rng.uniform(size=(H, W)) < rng.uniform(0.05, 0.3)), origin


def _carve(occ, origin, res, robots, radius):
    """Frees the cells within radius + res + 0.3 of every robot's start point (start bodies stay clear)."""
    H, W = occ.shape
    cx = origin[0] + (np.arange(W) + 0.5) * res
    cy = origin[1] + (np.arange(H) + 0.5) * res
    for rb in robots:
        d = np.hypot(cx[None, :] - rb["start"][0], cy[:, None] - rb["start"][1])
        occ[d <= radius + res + 0.3] = False
    return occ


def _map_scenes(B, K, seed, robots):
    """_mixed_fleet_scenes (circles, polygons, outlines, about half reactive) with a map in 7 of 8 environments: random noise
    (5..30 % occupied), a maze or a cave, at the resolutions 0.05, 0.1, 0.37 and 1 m, each carved clear around the robots' starts."""
    scenes = _mixed_fleet_scenes(B, K, seed, robots)
    radius = max(max(math.hypot(*v) for v in np.asarray(r.vertices, np.float64).T) for r in robots)
    for b, sc in enumerate(scenes):
        if b % 8 == 7:
            continue
        rng = np.random.default_rng([seed, K, b, 99])
        res = RESOLUTIONS[b % 4]
        kind = (b // 4) % 3
        if kind == 0:
            occ, origin = _noise_map(rng, res)
        elif kind == 1:
            m = maze(1, cells=(4, 4), cell_size=6.0, wall=max(0.3, 1.5 * res), resolution=res, seed=seed * 1000 + b)[0]["map"]
            occ, origin = m["occupancy"].copy(), (-12.5, -12.5)
        else:
            coarse = res * max(1, int(round(1.0 / res)))
            m = cave(1, size=(24.0, 24.0), resolution=res, coarse=coarse, clearance=1.0, seed=seed * 1000 + b)[0]["map"]
            occ, origin = m["occupancy"].copy(), (-12.0, -12.0)
        robs = sc["robots"] if "robots" in sc else [sc]
        sc["map"] = dict(occupancy=_carve(occ, origin, res, robs, radius), origin=origin, resolution=res)
    return scenes


RUNS = {"diff_K1_R1080": (("diff",), 1, 1080), "acker_K4_R37": (("acker",), 4, 37), "omni_K16_R37": (("omni",), 16, 37),
        "mixed3_K4_R37": (("diff", "acker", "omni"), 4, 37)}


@pytest.mark.parametrize("run", list(RUNS))
def test_teacher_forced_maps_match_the_oracle(run):
    """50 random-action steps of B = 128 scenes with maps: before every step the oracle takes the device's state; then every beam's
    hit, its range (1 ulp of the float32 oracle), velocity (exact), every clearance (0 ulp), flag and state must agree, with no
    beam excused.  Reactive obstacles keep the reactive tests' excuse (a decision margin below 1e-12 involving a robot)."""
    names, K, R = RUNS[run]
    B, steps, window = 128, 50, 1.5
    robots = [_robot(n) for n in names]
    kins = [r.kinematics for r in robots]
    lidar = dict(LIDAR, number=R, scan_offset=(0.1, 0.05, 0.1))
    scenes = _map_scenes(B, K, 23, robots)
    packed, beh, fleet, rtype = pack_scenes_ex(scenes), pack_behaviors(scenes), pack_fleet(scenes), pack_robot_types(scenes)
    w = WorldBatch(B, robots if len(robots) > 1 else robots[0], lidar, 0.1)
    w.set_scenes(scenes, seed=13, map_window=window)
    assert (w.K, w.N) == (K, B * K)
    o = MapOracleWorld(_oracle_cfg(robots[0], lidar), packed, beh, seed=13, fleet=fleet, K=K, types=_types_of(robots), robot_type=rtype,
                       maps=pack_maps(scenes), window=window)
    rng = np.random.default_rng(17)
    map_hits = map_collisions = excused_obs = 0
    worst_state, wrong = 0.0, []
    nobs = np.repeat(np.diff(o.obs_begin), K)[:, None]
    for k in range(steps):
        s = _device(w)
        o.obs[:], o.states[:], o.collided[:], o.arrived[:], o.goal[:], o.draws[:] = (s["obs"], s["states"], s["collided"], s["arrived"],
                                                                                     s["goal"], s["draws"])
        ranges, vel, _, hit = (t.cpu().numpy() if torch.is_tensor(t) else t for t in w.scan(hit=True))
        r64, v64, h64, _, _ = o.scan()
        assert np.array_equal(hit, h64), (k, np.argwhere(hit != h64)[:5])
        assert (_ulps(ranges, r64.astype(np.float32)) <= 1).all(), k
        assert np.array_equal(vel, v64.astype(np.float32)), k
        map_hits += int((h64 == nobs + K).sum())
        act = _mixed_actions(rng, kins, rtype, s["states"], K)
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
        for b in bad_env:
            ok[b * K:(b + 1) * K] = False
        worst_state = max(worst_state, float(np.abs(d["states"] - o.states)[ok].max()))
        assert np.array_equal(col[ok], o.collided[ok]) and np.array_equal(arr[ok], o.arrived[ok]), k
        u = _ulps(clear, clear_o.astype(np.float32))[ok]
        assert (u == 0).all(), (k, np.flatnonzero(u > 0)[:5])
        map_collisions += int(((o.map_clear <= 0.0) & (s["collided"] == 0)).sum())
    record(f"world_map_teacher_forced_{run}", envs=B, robots=B * K, beams=B * K * R, steps=steps, map_hits=map_hits,
           robot_map_collisions=map_collisions, collided_at_end=int(o.collided.sum()), excused_obstacles=excused_obs,
           max_state_err=worst_state, mismatches=len(wrong))
    assert not wrong, wrong[:3]
    assert worst_state <= 1e-12
    assert map_hits > 0 and map_collisions > 0  # OBSERVED: both are reported above
    w.close()


# ---- 3. edge cases -------------------------------------------------------------------------------------------------------------

def _one(occ, origin, res, robots, obstacles=(), bounds=(-40.0, -40.0, 40.0, 40.0)):
    return dict(obstacles=list(obstacles), bounds=bounds, robots=[dict(start=s, goal=(99.0, 99.0), goal_threshold=0.1, path=None) for s in robots],
                map=dict(occupancy=occ, origin=origin, resolution=res))


def _pair(scenes, lidar, window=1.0, kin="diff"):
    rb = _robot(kin)
    w = WorldBatch(len(scenes), rb, lidar, 0.1)
    w.set_scenes(scenes, map_window=window)
    o = MapOracleWorld(_oracle_cfg(rb, lidar), pack_scenes_ex(scenes), fleet=pack_fleet(scenes), K=len(scenes[0]["robots"]),
                       maps=pack_maps(scenes), window=window)
    return w, o


def _agree(w, o, act, steps=1):
    """scan and step against the oracle, bit for bit; returns the last (ranges, hit, collided, clearance)."""
    for _ in range(steps):
        ranges, vel, hit = (t.cpu().numpy() for t in w.scan(hit=True) if torch.is_tensor(t))
        r64, v64, h64, _, _ = o.scan()
        assert np.array_equal(hit, h64), np.argwhere(hit != h64)[:5]
        assert (_ulps(ranges, r64.astype(np.float32)) <= 1).all() and np.array_equal(vel, v64.astype(np.float32))
        col, _, clear = (t.cpu().numpy() for t in w.step(torch.from_numpy(act).cuda()))
        c_o, _, clear_o = o.step(act)
        assert np.array_equal(col, c_o) and np.array_equal(clear, clear_o.astype(np.float32))
    return ranges, hit, col, clear


def test_outcomes_of_the_stated_rules():
    """Each rule with its stated outcome, against the oracle."""
    d1 = dict(LIDAR, number=1, angle_min=0.0, angle_max=0.0, range_max=30.0)  # one beam along the heading (exactly +x at heading 0)
    occ = np.zeros((8, 8), bool)
    occ[3, 5] = True  # cell (5, 3) = [5, 6] x [3, 4]
    diag = np.zeros((8, 8), bool)
    diag[3, 5] = diag[4, 4] = True  # cells (5, 3) and (4, 4) meet at the corner (5, 4)
    wall = np.zeros((8, 8), bool)
    wall[:, 7] = True  # x in [7, 8]
    sq = [[-0.5, -0.5], [0.5, -0.5], [0.5, 0.5], [-0.5, 0.5]]
    cases = {  # name: (occupancy, origin, start, obstacles, scan_offset, (expected hit, expected range or None))
        "grid_line_row_below_unseen": (occ, (0.0, 0.0), (-3.0, 4.0, 0.0), [], (0.0, 0.0, 0.0), (-1, None)),  # y = 4: row 4
        "grid_line_row_seen": (occ, (0.0, 0.0), (-3.0, 3.0, 0.0), [], (0.0, 0.0, 0.0), (1, 8.0)),  # y = 3: row 3, x = 5
        "axis_parallel": (occ, (0.0, 0.0), (-3.0, 3.5, 0.0), [], (0.0, 0.0, 0.0), (1, 8.0)),
        "outside_looking_in": (occ, (10.0, 10.0), (0.0, 13.5, 0.0), [], (0.0, 0.0, 0.0), (1, 15.0)),
        "outside_looking_away": (occ, (10.0, 10.0), (30.0, 13.5, 0.0), [], (0.0, 0.0, 0.0), (-1, None)),
        "outside_looking_back": (occ, (10.0, 10.0), (30.0, 13.5, math.pi), [], (0.0, 0.0, 0.0), (1, None)),
        "in_occupied_cell_sees_exit": (wall, (0.0, 0.0), (2.0, 4.5, 0.0), [], (5.5, 0.0, 0.0), (1, 0.5)),  # sensor at x = 7.5
        "obstacle_edge_on_face_wins": (wall, (0.0, 0.0), (0.0, 4.5, 0.0), [dict(center=(7.5, 4.5), vertices=sq)], (0.0, 0.0, 0.0), (0, 7.0)),
        "range_max_cut_off": (wall, (30.0, 0.0), (0.0, 4.5, 0.0), [], (0.0, 0.0, 0.0), (-1, 30.0)),
    }
    got = {}
    for name, (grid, origin, start, obs, off, (want_hit, want_r)) in cases.items():
        lidar = dict(d1, scan_offset=off)
        w, o = _pair([_one(grid, origin, 1.0, [start], obstacles=obs)], lidar)
        ranges, hit, _, _ = _agree(w, o, np.zeros((1, 2), np.float32))
        got[name] = (int(hit[0, 0]), float(ranges[0, 0]))
        assert hit[0, 0] == want_hit, (name, got[name])
        if want_r is not None:
            assert abs(ranges[0, 0] - want_r) < 1e-5, (name, got[name])
        w.close()
    # a beam through the corner between two diagonal occupied cells: from (3, 2) at 45 degrees the beam meets the corner (5, 4) of
    # cells (4, 4) and (5, 3) (it passes free cells before), a hit there
    lidar = dict(d1, angle_min=math.pi / 4, angle_max=math.pi / 4)
    w, o = _pair([_one(diag, (0.0, 0.0), 1.0, [(3.0 - 0.5, 2.0 - 0.5, 0.0)])], lidar)
    ranges, hit, _, _ = _agree(w, o, np.zeros((1, 2), np.float32))
    assert hit[0, 0] == 1 and ranges[0, 0] <= math.hypot(2.5, 2.5) + 1e-5
    got["corner_between_diagonal_cells"] = (int(hit[0, 0]), float(ranges[0, 0]))
    record("world_map_stated_rules", **{k: list(v) for k, v in got.items()})
    w.close()


def test_touching_a_cell_face_collides_and_a_wall_beyond_the_window_reads_window():
    d1 = dict(LIDAR, number=1, angle_min=0.0, angle_max=0.0, range_max=30.0)
    rb = _robot("diff")
    front = max(v[0] for v in np.asarray(rb.vertices, np.float64).T)
    x_after = 1.0 + float(np.float32(5.0)) * 0.1  # the state after one step at 5 m/s, heading 0
    face = x_after + front
    r = 0.5
    occ = np.zeros((16, 8), bool)
    occ[:, 4] = True  # cell column 4: [x0 + 2, x0 + 2.5]
    w, o = _pair([_one(occ, (face - 2.0, -4.0), r, [(1.0, 0.0, 0.0)])], d1)
    _, _, col, clear = _agree(w, o, np.array([[5.0, 0.0]], np.float32))
    assert col[0] == 1 and clear[0] == 0.0  # the front edge lies on the face after the step: collided
    w.close()
    window = 1.25
    w, o = _pair([_one(occ, (1.0 + front + window + 0.05 - 2.0, -4.0), r, [(1.0, 0.0, 0.0)])], d1, window=window)
    _, _, col, clear = _agree(w, o, np.zeros((1, 2), np.float32), steps=2)
    assert col[0] == 0 and clear[0] == np.float32(window)  # the wall 0.05 m past the window: clearance == window
    w.close()


def test_a_full_size_map_and_two_handles_in_turn():
    """An 8192 x 8192 map (0.01 m cells, sparse walls), and a map-free handle used between its calls: both against what they must be."""
    N = 8192
    occ = np.zeros((N, N), bool)
    occ[4000:4100, 5000] = True
    occ[4050, 4200:4400] = True
    lidar = dict(LIDAR, number=360, range_max=30.0)
    sc = _one(occ, (-40.96, -40.96), 0.01, [(-1.0, -0.1, 0.3)])
    w, o = _pair([sc], lidar, window=0.5)
    plain_scenes = dyna_non_obs(8, seed=4)
    p1, p2 = WorldBatch(8, _robot("diff"), lidar, 0.1), WorldBatch(8, _robot("diff"), lidar, 0.1)
    p1.set_scenes(plain_scenes)
    p2.set_scenes(plain_scenes)
    act = np.array([[1.5, 0.1]], np.float32)
    pact = torch.full((8, 2), 0.5, device="cuda")
    for _ in range(10):
        ranges, hit, _, _ = _agree(w, o, act)
        a = _outputs(p1, pact)  # between the map handle's calls
        b = _outputs(p2, pact)
        assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert (hit == 1).any()
    record("world_map_8192", map_hits=int((hit == 1).sum()))
    for x in (w, p1, p2):
        x.close()


# ---- 4. closed loop --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("scene", ["maze", "cave"])
def test_closed_loop_maze_and_cave(scene):
    """C4's diff planner with its adjust values and the 100-beam lidar over pi in 128 maze or cave environments, with scans and
    blind; two rollouts with scans are bit-identical and a rollout does not synchronise the host."""
    steps = 200
    scenes = maze(128, seed=2024) if scene == "maze" else cave(128, seed=2024)
    seen, blind, again = _closed_loop(scenes, steps), _closed_loop(scenes, steps, blind=True), _closed_loop(scenes, steps)
    for k in ("states", "collided", "arrived", "steps_to_arrive", "min_clearance"):
        assert np.array_equal(seen[k], again[k]), k
    record(f"world_map_closed_loop_{scene}", envs=128, steps=steps, arrived_with_scans=int(seen["arrived"].sum()),
           collided_with_scans=int(seen["collided"].sum()), arrived_blind=int(blind["arrived"].sum()),
           collided_blind=int(blind["collided"].sum()), min_clearance_median=float(np.median(seen["min_clearance"])))
    pl = _planner(16, EXAMPLE_LIDAR)
    pl.set_initial_paths([sc["path"] for sc in scenes[:16]])
    w = WorldBatch(16, pl.robot, EXAMPLE_LIDAR, pl.dt)
    w.set_scenes(scenes[:16])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        rollout(pl, w, 5)
        rollout(pl, w, 5, blind=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    pl.close(); w.close()
