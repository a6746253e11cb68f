"""Mixed fleets in the batched world on the GPU: every robot type 0 through nb_world_set_fleet_ex against nb_world_set_fleet
(bitwise, the same launches), a K = 1 world of per-environment types against three single-type worlds (bitwise), teacher-forced
parity against the float64 oracle (tests/world_mixed_oracle.py) for K in {3, 8, 16} and mixes of 2, 3 and 4 types, edge cases, MixedPlanner, and a closed-loop
mixed_swap of diff, acker and omni planners."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from gpu_helpers import record
from helpers import CONFIGS, weights_path
from neupan_b200 import MixedPlanner, PlannerBatch, WorldBatch, _lib, rollout
from neupan_b200.robot import robot as Robot
from neupan_b200.world import (EXAMPLE_RVO, dyna_non_obs, make_robot_type, mixed_swap, pack_behaviors, pack_fleet, pack_robot_types,
                               pack_scenes_ex, random_outline, scene_paths)
from oracle import world as ow
from oracle.world import clearance_robot_pairs, clearance_robots
from test_gpu_world import EXAMPLE_LIDAR, LIDAR, _oracle_cfg, _polygon, _ulps
from test_gpu_world_fleet import _actions, _device, _fleet_scenes
from test_gpu_world_outline import _StillPlanner
from test_gpu_world_rvo import ROBOT_KW, _behavior
from world_mixed_oracle import MixedOracleWorld

pytestmark = pytest.mark.gpu

OCTAGON = [[1.2 * math.cos(k * math.pi / 4), 0.9 * math.sin(k * math.pi / 4)] for k in range(8)]
TRIANGLE = [[-0.9, -0.7], [1.1, 0.0], [-0.9, 0.7]]
# the robot types of each mix: type 0 is the config's robot (C4's diff body); then C2's car, C5's trapezoid (omni), and an octagonal
# acker robot with a short wheelbase
MIXES = {"diff_acker": ("diff", "acker"), "diff_acker_omni": ("diff", "acker", "omni"), "four": ("diff", "acker", "omni", "octagon")}


def _robot(name):
    if name == "octagon":
        return Robot(10, 0.1, kinematics="acker", vertices=OCTAGON, wheelbase=1.5)
    if name == "triangle":
        return Robot(10, 0.1, kinematics="omni", vertices=TRIANGLE)
    return Robot(10, 0.1, **ROBOT_KW[name])


def _types_of(robots):
    """The oracle's type dicts of robot types 1..T."""
    return [dict(kinematics=r.kinematics, wheelbase=r.L, robot_vertices=np.asarray(r.vertices, np.float64).T) for r in robots[1:]]


def _set_fleet_ex(w, robots, K, rows, rtype):
    rows = np.ascontiguousarray(np.asarray(rows, np.float64).reshape(-1, 6))
    rtype = np.ascontiguousarray(rtype, np.int32)
    types = (_lib.WorldRobotType * max(1, len(robots) - 1))(*[make_robot_type(r) for r in robots[1:]])
    with torch.cuda.device(w.device):
        _lib.check(_lib.load().nb_world_set_fleet_ex(w._handle, len(robots) - 1, types, w.B, K, C.c_void_p(rows.ctypes.data),
                                                     C.c_void_p(rtype.ctypes.data)))
    w.K, w.N = K, w.B * K


def _mixed_actions(rng, kins, rtype, states, K):
    """_actions of the fleet tests for each kinematics, each robot taking its own type's."""
    per = {k: _actions(rng, k, states, K) for k in sorted(set(kins))}
    return np.stack([per[kins[t]][n] for n, t in enumerate(rtype)]).astype(np.float32)


def _outputs(w, act):
    a = [t for t in w.scan(hit=True) if torch.is_tensor(t)] + list(w.step(act))
    return a + [w.states, w.obstacles()] + list(w.flags())


# ---- 1. every robot type 0 through _ex is the plain fleet ------------------------------------------------------------------

@pytest.mark.parametrize("reactive", [False, True])
def test_all_type_zero_through_ex_is_the_plain_fleet(reactive):
    B, K = 64, 5
    robots = [_robot("diff"), _robot("acker"), _robot("omni")]
    lidar = dict(LIDAR, number=90, scan_offset=(0.2, -0.1, 0.05))
    scenes = _fleet_scenes(B, K, 31, robots[0])
    if not reactive:
        scenes = [dict(sc, obstacles=[{k: v for k, v in ob.items() if k != "behavior"} for ob in sc["obstacles"]]) for sc in scenes]
    plain, ex = WorldBatch(B, robots[0], lidar, 0.1), WorldBatch(B, robots[0], lidar, 0.1)
    plain.set_scenes(scenes, seed=7)
    ex.set_scenes(scenes, seed=7)
    _set_fleet_ex(ex, robots, K, pack_fleet(scenes), np.zeros(B * K, np.int32))
    lib = _lib.load()
    rng = np.random.default_rng(8)
    for _ in range(50):
        act = torch.from_numpy(_actions(rng, "diff", plain.states.cpu().numpy(), K)).cuda()
        n0 = lib.nb_launch_count()
        a = _outputs(plain, act)
        n1 = lib.nb_launch_count()
        b = _outputs(ex, act)
        n2 = lib.nb_launch_count()
        assert n1 - n0 == n2 - n1 == (3 if reactive else 2)
        assert all(torch.equal(x, y) for x, y in zip(a, b))
    if reactive:
        assert all(torch.equal(x, y) for x, y in zip(plain.goals(), ex.goals()))
    c, _ = plain.flags()
    record(f"world_mixed_type_zero_ex_reactive{int(reactive)}", envs=B, robots=B * K, steps=50, collided=int(c.sum()))
    plain.close(); ex.close()


# ---- 2. K = 1, per-environment types: three single-type worlds -------------------------------------------------------------

def _kind_actions(rng, kin, n):
    if kin == "omni":
        return np.column_stack([rng.uniform(-1.5, 1.5, n), rng.uniform(-1.5, 1.5, n)]).astype(np.float32)
    return np.column_stack([rng.uniform(-1.0, 2.0, n), rng.uniform(-0.5, 0.5, n)]).astype(np.float32)


@pytest.mark.parametrize("reactive", [False, True])
def test_per_environment_types_equal_single_type_worlds(reactive):
    """3B environments of one seeded scene set, environment b of type b mod 3 (diff, acker, polygon omni), against three worlds of
    one type on environments t, t + 3, ...: every scan, step, state, obstacle row and flag, bit for bit, over 50 random steps.
    Reactive obstacles head for explicit goals (no wander: goal draws are keyed by the environment index)."""
    B = 40
    names = ("diff", "acker", "omni")
    robots = [_robot(n) for n in names]
    lidar = dict(LIDAR, number=120, scan_offset=(0.1, 0.05, 0.0))
    scenes = dyna_non_obs(3 * B, seed=9)
    rng = np.random.default_rng(10)
    for b, sc in enumerate(scenes):
        sc["type"] = b % 3
        if reactive:
            sc["obstacles"] = [dict(ob, velocity=(0.0, 0.0), behavior=dict(EXAMPLE_RVO, wander=False, goal=tuple(rng.uniform((6.0, 16.0), (44.0, 34.0)))))
                               for ob in sc["obstacles"]]
    mixed = WorldBatch(3 * B, robots, lidar, 0.1)
    mixed.set_scenes(scenes, seed=3)
    assert mixed.K == 1 and mixed.robot_types.tolist() == [b % 3 for b in range(3 * B)]
    singles = []
    for t in range(3):
        w = WorldBatch(B, robots[t], lidar, 0.1)
        w.set_scenes([{k: v for k, v in sc.items() if k != "type"} for sc in scenes[t::3]], seed=3)
        singles.append(w)
    O = np.concatenate([[0], np.cumsum([len(sc["obstacles"]) for sc in scenes])])
    obs_rows = [np.concatenate([np.arange(O[b], O[b + 1]) for b in range(t, 3 * B, 3)]) for t in range(3)]
    obs_rows = [torch.from_numpy(r).cuda() for r in obs_rows]
    hits = 0
    for _ in range(50):
        acts = [torch.from_numpy(_kind_actions(rng, names[t], B)).cuda() for t in range(3)]
        act = torch.empty((3 * B, 2), device="cuda")
        for t in range(3):
            act[t::3] = acts[t]
        m = [t for t in mixed.scan(hit=True) if torch.is_tensor(t)] + list(mixed.step(act)) + [mixed.states] + list(mixed.flags())
        m_obs = mixed.obstacles()
        for t, w in enumerate(singles):
            s = [x for x in w.scan(hit=True) if torch.is_tensor(x)] + list(w.step(acts[t])) + [w.states] + list(w.flags())
            assert all(torch.equal(x[t::3], y) for x, y in zip(m, s)), t
            assert torch.equal(m_obs.index_select(0, obs_rows[t]), w.obstacles()), t
            if reactive:
                assert torch.equal(mixed.goals()[0].index_select(0, obs_rows[t]), w.goals()[0]), t
        hits += int((m[2] >= 0).sum())
    c, a = mixed.flags()
    record(f"world_mixed_per_env_types_reactive{int(reactive)}", envs=3 * B, steps=50, beam_hits=hits,
           collided_per_type=[int(c[t::3].sum()) for t in range(3)])
    assert hits > 0
    for w in [mixed] + singles:
        w.close()


# ---- 3. teacher-forced parity --------------------------------------------------------------------------------------------------

def _mixed_fleet_scenes(B, K, seed, robots):
    """Mixed obstacles (about half reactive) in [-12, 12]^2 and K robots of random types placed at random in [-8, 8]^2, start
    bodies (each its own type's polygon) at least 0.3 m apart."""
    verts = [np.asarray(r.vertices, np.float64).T for r in robots]
    scenes = []
    for b in range(B):
        rng = np.random.default_rng([seed, K, len(robots), b])
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
        fleet, bodies = [], []
        while len(fleet) < K:
            # the first min(K, T + 1) robots take distinct types (every type appears somewhere), the others random ones
            t = (b + len(fleet)) % len(robots) if len(fleet) < len(robots) else int(rng.integers(0, len(robots)))
            s = (rng.uniform(-8, 8), rng.uniform(-8, 8), rng.uniform(-np.pi, np.pi))
            body = ow.robot_polygon(s, verts[t])
            if any(clearance_robots(body, q) < 0.3 for q in bodies):
                continue
            bodies.append(body)
            fleet.append(dict(start=s, goal=tuple(rng.uniform(-8, 8, 2)), goal_threshold=rng.uniform(0.3, 1.0), path=None, type=t))
        order = rng.permutation(K)
        scenes.append(dict(obstacles=obs, bounds=(-12.0, -12.0, 12.0, 12.0), robots=[fleet[i] for i in order]))
    return scenes


@pytest.mark.parametrize("mix", list(MIXES))
@pytest.mark.parametrize("K", [3, 8, 16])
def test_teacher_forced_mixed_fleet_matches_the_oracle(K, mix):
    """The bars of test_gpu_world_fleet's teacher-forced test, with a mix of robot types in every environment."""
    B, steps = 128, 50
    names = MIXES[mix]
    robots = [_robot(n) for n in names]
    kins = [r.kinematics for r in robots]
    lidar = dict(LIDAR, number=16, scan_offset=(0.1, 0.05, 0.1))
    scenes = _mixed_fleet_scenes(B, K, 71, robots)
    packed, beh, fleet, rtype = pack_scenes_ex(scenes), pack_behaviors(scenes), pack_fleet(scenes), pack_robot_types(scenes)
    w = WorldBatch(B, robots, lidar, 0.1)
    w.set_scenes(scenes, seed=13)
    assert (w.K, w.N) == (K, B * K) and np.array_equal(w.robot_types, rtype)
    assert all(np.array_equal(w.rows_of_type(t).cpu().numpy(), np.flatnonzero(rtype == t)) for t in range(len(robots)))
    o = MixedOracleWorld(_oracle_cfg(robots[0], lidar), packed, beh, seed=13, fleet=fleet, K=K, types=_types_of(robots), robot_type=rtype)
    rng = np.random.default_rng(17)
    robot_hits = excused_beams = excused_obs = worst_state = ulp1 = 0
    pair_hits, pair_collisions = {}, {}
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
        rh = np.argwhere(h64 >= nobs)
        robot_hits += len(rh)
        for n, i in rh:  # (seeing type, seen type)
            key = f"{names[rtype[n]]}>{names[rtype[(n // K) * K + h64[n, i] - nobs[n, 0]]]}"
            pair_hits[key] = pair_hits.get(key, 0) + 1
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
        assert np.array_equal(d["collided"], col) and np.array_equal(d["arrived"], arr)
        u = _ulps(clear, clear_o.astype(np.float32))[ok]
        assert (u <= 1).all(), (k, np.flatnonzero(u > 1)[:5])
        ulp1 += int((u == 1).sum())
        for n in np.flatnonzero((o.robot_clear <= 0.0) & (s["collided"] == 0)):  # new robot-robot collisions, by type pair
            b = n // K
            bodies = o.bodies(b)
            for j in range(K):
                if b * K + j != n and clearance_robots(bodies[n - b * K], bodies[j]) <= 0.0:
                    key = "+".join(sorted((names[rtype[n]], names[rtype[b * K + j]])))
                    pair_collisions[key] = pair_collisions.get(key, 0) + 1
    record(f"world_mixed_teacher_forced_{mix}_K{K}", envs=B, robots=B * K, steps=steps, robot_hits=robot_hits, robot_hits_by_pair=pair_hits,
           robot_robot_collisions_by_pair=pair_collisions, collided_at_end=int(o.collided.sum()), excused_beams=excused_beams,
           excused_obstacles=excused_obs, max_state_err=worst_state, clearance_ulp1=ulp1, mismatches=len(wrong))
    assert not wrong, wrong[:3]
    assert worst_state <= 1e-12
    assert robot_hits > 0 and sum(pair_collisions.values()) > 0  # OBSERVED: both are reported above
    assert any("+" in k and k.split("+")[0] != k.split("+")[1] for k in pair_collisions)  # robots of different types collided
    w.close()


# ---- 4. edge cases ---------------------------------------------------------------------------------------------------------

def _check_against_oracle(w, o, act, steps):
    """scan and step against the oracle for ``steps`` steps of the constant action; returns the per-step collided flags."""
    cols = []
    for _ in range(steps):
        ranges, vel, hit = (t.cpu().numpy() for t in w.scan(hit=True) if torch.is_tensor(t))
        r64, v64, h64, _, _ = o.scan()
        assert np.array_equal(hit, h64) and (_ulps(ranges, r64.astype(np.float32)) <= 1).all() and np.array_equal(vel, v64.astype(np.float32))
        col, _, clear = (t.cpu().numpy() for t in w.step(torch.from_numpy(act).cuda()))
        c_o, _, clear_o = o.step(act)
        assert np.array_equal(col, c_o) and (_ulps(clear, clear_o.astype(np.float32)) <= 1).all()
        cols.append(col.copy())
    return np.array(cols)


def _scene(robots, obstacles=()):
    return dict(obstacles=list(obstacles), bounds=(-30.0, -30.0, 30.0, 30.0),
                robots=[dict(start=s, goal=(50.0, 50.0), goal_threshold=0.1, path=None, type=t) for s, t in robots])


def _world(robots, scenes, lidar):
    w = WorldBatch(len(scenes), robots, lidar, 0.1)
    w.set_scenes(scenes)
    o = MixedOracleWorld(_oracle_cfg(robots[0], lidar), pack_scenes_ex(scenes), fleet=pack_fleet(scenes), K=len(scenes[0]["robots"]),
                    types=_types_of(robots), robot_type=pack_robot_types(scenes))
    return w, o


def test_a_car_and_an_omni_robot_head_on_collide_in_the_same_step():
    robots = [_robot("diff"), _robot("acker"), _robot("omni")]
    lidar = dict(LIDAR, number=9, range_max=20.0)
    # the car (type 1) heads +x from its rear axle at x = 0; the trapezoid (type 2) sits 12 m ahead, sliding -x; a diff robot far off
    sc = _scene([((0.0, 0.0, 0.0), 1), ((12.0, 0.0, 0.0), 2), ((0.0, 20.0, 0.0), 0)])
    w, o = _world(robots, [sc], lidar)
    act = np.array([[2.0, 0.0], [-1.5, 0.0], [0.0, 0.0]], np.float32)
    cols = _check_against_oracle(w, o, act, 40)
    first = np.argmax(cols.any(1))
    assert cols[:, :2].any() and cols[first, 0] == cols[first, 1] == 1 and cols[first, 2] == 0  # both in the same step
    record("world_mixed_car_omni_head_on", collided_at_step=int(first) + 1)
    w.close()


def test_a_robot_hit_reports_the_hit_robots_own_velocity():
    """Robot 0 (diff) looks along +x at a car and, behind it, along -x at an omni robot: after one step the beams report the car's
    v (cos th, sin th) and the omni robot's (vx, vy)."""
    robots = [_robot("diff"), _robot("acker"), _robot("omni")]
    lidar = dict(LIDAR, number=2, angle_min=0.0, angle_max=math.pi, range_max=25.0)  # beams along +x and -x
    th = 0.3
    sc = _scene([((0.0, 0.0, 0.0), 0), ((8.0, -1.0, th), 1), ((-8.0, 0.0, 0.0), 2)])
    w, o = _world(robots, [sc], lidar)
    act = np.array([[0.0, 0.0], [1.5, 0.2], [0.25, -0.5]], np.float32)
    _check_against_oracle(w, o, act, 1)
    _, vel, _, hit = w.scan(hit=True)
    assert hit[0].tolist() == [1, 2]  # no obstacles: robot j is hit index j
    v = vel[0].cpu().numpy()
    assert v[:, 1].tolist() == [0.25, -0.5]
    assert abs(v[0, 0] - 1.5 * math.cos(th)) < 1e-6 and abs(v[1, 0] - 1.5 * math.sin(th)) < 1e-6  # the car's heading before the step
    r64, v64, h64, _, _ = o.scan()
    assert np.array_equal(v, v64.astype(np.float32)[0])
    w.close()


def test_three_and_eight_vertex_types_see_and_are_seen():
    """A 3-vertex omni type and an 8-vertex acker type beside the 4-vertex config robot: their bodies are what the beams cross and
    what the clearances are taken from, against the oracle, for several environments and headings; they drive into each other."""
    robots = [_robot("diff"), _robot("triangle"), _robot("octagon")]
    lidar = dict(LIDAR, number=360, range_max=15.0, scan_offset=(0.3, 0.0, 0.0))
    scenes = []
    for b in range(24):
        a = 0.26 * b
        scenes.append(_scene([((0.0, 0.0, a), 0), ((4.0 * math.cos(a), 4.0 * math.sin(a), a + 2.0), 1),
                              ((-4.5 * math.cos(a + 0.4), -4.5 * math.sin(a + 0.4), a - 1.0), 2)],
                             [dict(center=(9.0, 9.0), radius=0.8), dict(center=(-9.0, 5.0), vertices=[[-1, -1], [1, -1], [1, 1], [-1, 1]])]))
    w, o = _world(robots, scenes, lidar)
    assert sorted({len(p) for b in range(24) for p in o.bodies(b)}) == [3, 4, 8]
    _, _, _, hit = w.scan(hit=True)
    hit = hit.cpu().numpy().reshape(24, 3, -1)
    for b in range(24):  # robot 0, between the others, sees both; they see robot 0 (it hides the other one from them)
        assert {3, 4} <= set(hit[b, 0].tolist()) and 2 in hit[b, 1] and 2 in hit[b, 2], b
    # robots 1 and 2 drive at robot 0
    act = np.zeros((72, 2), np.float32)
    for b in range(24):
        a = 0.26 * b
        act[3 * b + 1] = (-1.0 * math.cos(a), -1.0 * math.sin(a))  # omni: (vx, vy) towards the centre
        act[3 * b + 2] = (1.0, 0.0)
    cols = _check_against_oracle(w, o, act, 40)
    assert cols[-1].sum() >= 24
    record("world_mixed_three_eight_vertices", collided=int(cols[-1].sum()))
    w.close()


# ---- 5. MixedPlanner -----------------------------------------------------------------------------------------------------------

def _planner(cname, N, R):
    cfg = CONFIGS[cname]
    return PlannerBatch(N, cfg.T, cfg.dt, 4.0, robot_kwargs=cfg.robot_kwargs, adjust_kwargs=dict(cfg.adjust),
                        pan_kwargs=dict(iter_num=cfg.K, dune_max_num=R, nrmp_max_num=cfg.M, dune_checkpoint=weights_path(cfg.model),
                                        iter_threshold=0.0, max_points=R))


KINDS = ("C4", "C2", "C5")  # type 0: diff, 1: acker, 2: polygon omni, each config's adjust values and checkpoint


def _mixed_setup(scenes, R=EXAMPLE_LIDAR["number"]):
    rtype = pack_robot_types(scenes)
    pls = [_planner(c, int((rtype == t).sum()), R) for t, c in enumerate(KINDS)]
    w = WorldBatch(len(scenes), [p.robot for p in pls], EXAMPLE_LIDAR, pls[0].dt)
    w.set_scenes(scenes)
    for t, p in enumerate(pls):
        p.set_initial_paths(scene_paths(scenes, type=t))
    return w, pls, MixedPlanner([(p, w.rows_of_type(t)) for t, p in enumerate(pls)])


def test_mixed_planner_is_each_kinds_planner_on_its_rows():
    scenes = mixed_swap(16, robots=6, seed=4, circles=2)
    w, pls, mp = _mixed_setup(scenes)
    twins = [_planner(c, p.B, EXAMPLE_LIDAR["number"]) for c, p in zip(KINDS, pls)]
    for t, p in enumerate(twins):
        p.set_initial_paths(scene_paths(scenes, type=t))
    for _ in range(5):
        ranges, vel, scan = w.scan()
        states = w.states
        action, infos = mp.forward(states, ranges, scan, scan_offset=w.scan_offset, scan_velocity=vel)
        assert action.shape == (96, 2) and len(infos) == 3
        for t, p in enumerate(twins):
            rows = w.rows_of_type(t)
            a, _ = p.forward(states[rows], ranges[rows], scan, scan_offset=w.scan_offset, scan_velocity=vel[rows])
            assert torch.equal(action[rows], a), t
        w.step(action)
    assert w.rows_of_type(2).tolist() == [n for n in range(96) if n % 6 in (2, 5)]
    with pytest.raises(ValueError, match="exactly once"):
        MixedPlanner([(pls[0], w.rows_of_type(0)), (pls[1], w.rows_of_type(0))])
    for x in pls + twins:
        x.close()
    w.close()


def test_mixed_rollout_does_not_synchronise_the_host():
    B = 16
    robots = [_robot("diff"), _robot("acker"), _robot("omni")]
    w = WorldBatch(B, robots, EXAMPLE_LIDAR, 0.1)
    w.set_scenes(mixed_swap(B, robots=6, seed=1))

    class Still(_StillPlanner):
        def __init__(self, n):
            super().__init__(n)
            self.B, self.device = n, torch.device("cuda")

    mp = MixedPlanner([(Still(len(w.rows_of_type(t))), w.rows_of_type(t)) for t in range(3)])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = rollout(mp, w, 5)
        out = rollout(mp, w, 5, velocities=False)
        out = rollout(mp, w, 5, blind=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert out["min_clearance"].shape == (B * 6,)
    w.close()


# ---- 6. closed loop --------------------------------------------------------------------------------------------------------

SWAP_STEPS = 120


def _swap_loop(scenes, steps, **kw):
    w, pls, mp = _mixed_setup(scenes)
    out = rollout(mp, w, steps, **kw)
    out = {k: v.cpu().numpy() for k, v in out.items()}
    out["states"] = w.states.cpu().numpy()
    rtype = w.robot_types
    B, K = len(scenes), 6
    bodies = [ow.robot_polygon(s, np.asarray(w.robots[t].vertices, np.float64).T) for s, t in zip(out["states"], rtype)]
    rr = np.array([min(clearance_robots(bodies[n], bodies[(n // K) * K + j]) for j in range(K) if (n // K) * K + j != n) for n in range(B * K)])
    out["robot_robot"] = out["collided"] & (rr <= 0.0)
    out["type"] = rtype
    mp.close(); w.close()
    return out


def test_closed_loop_mixed_swap():
    scenes = mixed_swap(128, robots=6, seed=2024)
    legs = {"scans": _swap_loop(scenes, SWAP_STEPS), "blind": _swap_loop(scenes, SWAP_STEPS, blind=True)}
    again = _swap_loop(scenes, SWAP_STEPS)
    for k in ("states", "collided", "arrived", "steps_to_arrive", "min_clearance"):
        assert np.array_equal(legs["scans"][k], again[k]), k
    summary = {}
    for name, out in legs.items():
        for t, kind in enumerate(("diff_C4", "acker_C2", "omni_C5")):
            m = out["type"] == t
            arrived = out["steps_to_arrive"][m & out["arrived"]]
            summary[f"{name}_{kind}"] = dict(robots=int(m.sum()), arrived=int((m & out["arrived"]).sum()), collided=int((m & out["collided"]).sum()),
                                             collided_robot_robot=int((m & out["robot_robot"]).sum()),
                                             median_steps_to_arrive=float(np.median(arrived)) if len(arrived) else -1.0)
    record("world_mixed_closed_loop_mixed_swap", envs=128, robots=768, steps=SWAP_STEPS, **summary)
    # Observed on one H100 (256 robots of each kind, 120 steps), with scans: diff 72 arrived / 90 collided (median 80 steps), acker
    # 45 / 145 (64), omni 40 / 157 (66.5), every collision robot-robot; blind: all 768 collide and none arrives.  The thresholds sit
    # just below (above for collisions).
    for kind, arrived, collided in (("diff_C4", 65, 100), ("acker_C2", 40, 155), ("omni_C5", 35, 165)):
        assert summary[f"scans_{kind}"]["arrived"] >= arrived and summary[f"scans_{kind}"]["collided"] <= collided, kind
        assert summary[f"blind_{kind}"]["collided"] >= 250 and summary[f"blind_{kind}"]["arrived"] == 0, kind
