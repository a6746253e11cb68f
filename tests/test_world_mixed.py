"""Mixed fleets in the batched world, on the CPU: host validation through nb_world_check_fleet_ex, the packing of robot types, the
plain fleet calls as the _ex calls without types, the oracle's robot-robot clearance between different polygons and the mixed_swap
builder (no device needed)."""
import ctypes as C
import math

import numpy as np
import pytest

from neupan_b200 import _lib, build as nb_build
from neupan_b200.robot import robot as Robot
from neupan_b200.world import (circle_swap, make_config, make_robot_type, mixed_swap, pack_fleet, pack_robot_types, pack_scenes_ex,
                               scene_paths)
from oracle import world as ow
from oracle.world import clearance_robot_pairs, clearance_robots
from world_mixed_oracle import MixedOracleWorld

LIDAR = dict(angle_min=-math.pi, angle_max=math.pi, range_min=0.0, range_max=10.0, number=36)
# the three shipped bodies: C4's diff robot, C2's car, C5's trapezoid (omni)
DIFF = dict(kinematics="diff", length=1.6, width=2.0)
ACKER = dict(kinematics="acker", length=4.6, width=1.6, wheelbase=3)
OMNI = dict(kinematics="omni", vertices=[[-0.8, -1.0], [-1.8, 1.0], [1.8, 1.0], [0.8, -1.0]])


@pytest.fixture(scope="module")
def lib():
    nb_build.build()
    return _lib.load()


def _robots(*kws):
    return [Robot(10, 0.1, **kw) for kw in kws]


def _types(robots):
    return (_lib.WorldRobotType * max(1, len(robots)))(*[make_robot_type(r) for r in robots])


def _check_ex(lib, cfg, types, B, K, rows, rtype):
    rows = np.ascontiguousarray(np.asarray(rows, np.float64).reshape(-1, 6))
    rt = None if rtype is None else np.ascontiguousarray(rtype, np.int32)
    return lib.nb_world_check_fleet_ex(C.byref(cfg), len(types) if types is not None else 0, types, B, K, C.c_void_p(rows.ctypes.data),
                                       None if rt is None else C.c_void_p(rt.ctypes.data))


def test_host_validation_of_mixed_fleets(lib):
    diff, car, omni = _robots(DIFF, ACKER, OMNI)
    cfg = make_config(diff, LIDAR, 0.1, max_envs=4)
    types = _types([car, omni])
    rows = [[0.0, 0.0, 0.0, 5.0, 0.0, 0.3], [0.0, 5.0, 0.0, 5.0, 5.0, 0.3], [0.0, -5.0, 0.0, 5.0, -5.0, 0.3]]
    assert _check_ex(lib, cfg, types, 1, 3, rows, [0, 1, 2]) == _lib.NB_OK
    assert _check_ex(lib, cfg, types, 3, 1, rows, [2, 1, 0]) == _lib.NB_OK  # K = 1: one robot per environment, of any type
    assert _check_ex(lib, cfg, None, 1, 3, rows, None) == _lib.NB_OK

    def refused(rc, msg):
        assert rc == _lib.NB_ERR_INVALID
        assert msg in lib.nb_last_error().decode(), lib.nb_last_error().decode()

    def bad_type(msg, **fields):
        t = _types([car, omni])
        for k, v in fields.items():
            if k == "vertices":
                t[1].vertices = (C.c_double * 16)(*(list(v) + [0.0] * (16 - len(v))))
            else:
                setattr(t[1], k, v)
        refused(_check_ex(lib, cfg, t, 1, 3, rows, [0, 1, 2]), msg)

    bad_type("robot type 2: kinematics 3 (diff, acker or omni)", kinematics=3)
    bad_type("robot type 2: kinematics -1 (diff, acker or omni)", kinematics=-1)
    bad_type("robot type 2: acker needs a positive wheelbase", kinematics=1, wheelbase=0.0)
    bad_type("robot type 2: acker needs a positive wheelbase", kinematics=1, wheelbase=-3.0)
    bad_type("robot type 2: the polygon needs 3..8 vertices (got 2)", num_vertices=2)
    bad_type("robot type 2: the polygon needs 3..8 vertices (got 9)", num_vertices=9)
    bad_type("robot type 2: the polygon is not convex", num_vertices=4, vertices=[-1, -1, 1, 1, 1, -1, -1, 1])  # a bow tie
    bad_type("robot type 2: the polygon is not convex", num_vertices=4, vertices=[-1, -1, 0, -0.5, 1, -1, 0, 1])  # a reflex corner
    bad_type("robot type 2: the polygon is not convex", num_vertices=3, vertices=[0, 0, math.nan, 0, 0, 1])
    t = _types([car])
    t[0].wheelbase = 0.0  # acker only: a wheelbase of 0 is fine for a diff type
    t[0].kinematics = 0
    assert _check_ex(lib, cfg, t, 1, 3, rows, [0, 1, 1]) == _lib.NB_OK
    refused(_check_ex(lib, cfg, types, 1, 3, rows, [0, 1, 3]), "environment 0, robot 2: type 3 outside 0..2")
    refused(_check_ex(lib, cfg, types, 1, 3, rows, [0, -1, 2]), "environment 0, robot 1: type -1 outside 0..2")
    refused(_check_ex(lib, cfg, None, 3, 1, rows, [0, 0, 1]), "environment 2, robot 0: type 1 outside 0..0")
    refused(_check_ex(lib, cfg, _types([car, omni, diff, car]), 1, 3, rows, [0, 1, 2]), "T = 4 robot types besides type 0 (0..3)")
    assert _check_ex(lib, cfg, _types([car, omni, diff]), 1, 3, rows, [0, 3, 2]) == _lib.NB_OK  # 4 types: the limit
    rr = np.ascontiguousarray(rows, np.float64)
    refused(lib.nb_world_check_fleet_ex(C.byref(cfg), 2, None, 1, 3, C.c_void_p(rr.ctypes.data), None), "nb_world fleet: null types")
    # overlap with each robot's own polygon: the car (x in -0.8 .. 3.8 about its rear axle) reaches a diff robot 4 m ahead, which a
    # diff robot in its place would not
    ahead = [[0.0, 0.0, 0.0, 9.0, 0.0, 0.3], [4.0, 0.0, 0.0, 9.0, 0.0, 0.3]]
    assert _check_ex(lib, cfg, types, 1, 2, ahead, [0, 0]) == _lib.NB_OK
    assert _check_ex(lib, cfg, types, 1, 2, ahead, [1, 1]) == _lib.NB_ERR_INVALID
    refused(_check_ex(lib, cfg, types, 1, 2, ahead, [1, 0]), "environment 0: the start bodies of robots 0 and 1 overlap")
    assert _check_ex(lib, cfg, types, 1, 2, ahead, [0, 1]) == _lib.NB_OK  # the car behind the diff robot points away from it
    # the trapezoid's wide side (y = 1, |x| <= 1.8) touches a diff robot above it exactly
    touch = [[0.0, 0.0, 0.0, 9.0, 0.0, 0.3], [0.0, 2.0, 0.0, 9.0, 2.0, 0.3]]
    refused(_check_ex(lib, cfg, types, 1, 2, touch, [2, 0]), "environment 0: the start bodies of robots 0 and 1 overlap")
    # a config check still comes first
    cfg_bad = make_config(diff, LIDAR, 0.1, max_envs=4)
    cfg_bad.robot_num_vertices = 2
    refused(_check_ex(lib, cfg_bad, types, 1, 3, rows, [0, 1, 2]), "the robot polygon needs 3..8 vertices")


def test_plain_fleet_check_is_the_ex_check_without_types(lib):
    """nb_world_check_fleet is nb_world_check_fleet_ex(T = 0, robot_type = NULL): the same verdict and message on every input."""
    diff, car = _robots(DIFF, ACKER)
    cfg = make_config(diff, LIDAR, 0.1, max_envs=4)
    ok = [[0.0, 0.0, 0.0, 5.0, 0.0, 0.3], [0.0, 3.0, 0.0, 5.0, 3.0, 0.3]]
    cases = [(1, 2, ok), (2, 2, ok + ok), (1, 1, ok[:1]), (1, 0, ok), (1, 17, [[4.0 * k, 0, 0, 0, 0, 0.3] for k in range(17)]),
             (5, 1, ok * 3), (2, 2, ok + [ok[0], [0.0, math.nan, 0.0, 5.0, 3.0, 0.3]]), (2, 2, ok + [ok[0], [0.0, 3.0, 0.0, 5.0, 3.0, -0.1]]),
             (1, 2, [ok[0], [0.0, 2.0, 0.0, 5.0, 3.0, 0.3]]), (1, 3, ok + [[0.0, 0.0, 1.0, 1.0, 1.0, 0.0]])]
    for B, K, rows in cases:
        rows = np.ascontiguousarray(np.asarray(rows, np.float64).reshape(-1, 6))
        rc = lib.nb_world_check_fleet(C.byref(cfg), B, K, C.c_void_p(rows.ctypes.data))
        msg = lib.nb_last_error().decode() if rc else ""
        rc_ex = lib.nb_world_check_fleet_ex(C.byref(cfg), 0, None, B, K, C.c_void_p(rows.ctypes.data), None)
        assert rc == rc_ex and (not rc or lib.nb_last_error().decode() == msg), (B, K, msg)
        zeros = np.zeros(B * max(K, 0), np.int32)
        rc_z = lib.nb_world_check_fleet_ex(C.byref(cfg), 1, _types([car]), B, K, C.c_void_p(rows.ctypes.data), C.c_void_p(zeros.ctypes.data))
        assert rc_z == rc and (not rc or lib.nb_last_error().decode() == msg), (B, K, msg)  # every robot type 0: the same checks


def _scene(robots, obstacles=()):
    return dict(obstacles=list(obstacles), bounds=(-20.0, -20.0, 20.0, 20.0),
                robots=[dict(start=s, goal=(5.0, 0.0), goal_threshold=0.3, path=np.array([[s[0], s[1], s[2], 1.0]]), **({} if t is None else {"type": t}))
                        for s, t in robots])


def test_packing_of_robot_types():
    a = _scene([((0.0, 0.0, 0.0), 1), ((0.0, 5.0, 0.0), None), ((0.0, -5.0, 0.0), 2)])
    b = _scene([((1.0, 0.0, 0.0), 2), ((1.0, 5.0, 0.0), 2), ((1.0, -5.0, 0.0), 0)])
    t = pack_robot_types([a, b])
    assert t.dtype == np.int32 and t.flags.c_contiguous and t.tolist() == [1, 0, 2, 2, 2, 0]
    assert pack_fleet([a, b]).shape == (6, 6)  # unchanged by the types
    assert [p[0, 0] for p in scene_paths([a, b], type=2)] == [0.0, 1.0, 1.0]  # row order: rows 2, 3, 4
    assert [p[0, 1] for p in scene_paths([a, b], type=0)] == [5.0, -5.0]
    assert len(scene_paths([a, b])) == 6 and scene_paths([a, b], type=3) == []
    single = dict(obstacles=[], bounds=(-1.0, -1.0, 1.0, 1.0), start=(0.0, 0.0, 0.0), goal=(1.0, 0.0), goal_threshold=0.5, path=None)
    assert pack_robot_types([single, dict(single, type=2)]).tolist() == [0, 2]
    assert pack_robot_types(circle_swap(3, robots=4)).tolist() == [0] * 12


def _random_polygon(rng):
    n = int(rng.integers(3, 9))
    ang = np.sort(rng.uniform(0, 2 * np.pi - 0.01, n)) + np.arange(n) * 1e-3
    return np.stack([rng.uniform(0.5, 2.5) * np.cos(ang), rng.uniform(0.5, 2.5) * np.sin(ang)], 1)


def test_oracle_robot_clearance_is_symmetric_between_different_polygons():
    rng = np.random.default_rng(3)
    shipped = [np.asarray(r.vertices, np.float64).T for r in _robots(DIFF, ACKER, OMNI)]
    pq, qp, pairs = [], [], []
    for m in range(3000):
        pa = shipped[m % 3] if m % 2 else _random_polygon(rng)
        pb = shipped[(m // 2) % 3] if m % 3 else _random_polygon(rng)
        s = (rng.uniform(-1, 1), rng.uniform(-1, 1), rng.uniform(-math.pi, math.pi))
        d, a = rng.uniform(0.0, 6.0), rng.uniform(-math.pi, math.pi)
        t = (s[0] + d * math.cos(a), s[1] + d * math.sin(a), rng.uniform(-math.pi, math.pi))
        P, Q = ow.robot_polygon(s, pa), ow.robot_polygon(t, pb)
        pq.append(clearance_robots(P, Q))
        qp.append(clearance_robots(Q, P))
        pairs.append((P, Q))
    pq, qp = np.array(pq), np.array(qp)
    assert np.array_equal(pq, qp)  # bit for bit
    assert (pq == 0.0).sum() > 300 and (pq > 0.0).sum() > 1000
    # the vectorised form the oracle uses per (vertex count, vertex count) class gives the same values
    for P, Q in pairs[:300]:
        P, Q = np.asarray(P)[None], np.asarray(Q)[None]
        assert clearance_robot_pairs(P, Q)[0] == clearance_robot_pairs(Q, P)[0] == clearance_robots([tuple(v) for v in P[0]], [tuple(v) for v in Q[0]])


def test_oracle_robot_clearances_group_mixed_vertex_counts():
    """MixedOracleWorld.robot_clearances over a mixed environment equals the pairwise minimum of clearance_robots."""
    diff, car, omni = _robots(DIFF, ACKER, OMNI)
    scenes = mixed_swap(4, types=(0, 1, 2, 3), robots=7, radius=7.0, seed=5)
    tri = [[-1.0, -1.0], [1.5, 0.0], [-1.0, 1.0]]
    cfg = dict(kinematics="diff", step_time=0.1, wheelbase=None, angle_min=-1.0, angle_max=1.0, range_max=5.0, number=3,
               scan_offset=(0.0, 0.0, 0.0), robot_vertices=np.asarray(diff.vertices, np.float64).T)
    types = [dict(kinematics=r.kinematics, wheelbase=r.L, robot_vertices=np.asarray(r.vertices, np.float64).T) for r in (car, omni)]
    types.append(dict(kinematics="omni", wheelbase=None, robot_vertices=np.asarray(tri)))
    o = MixedOracleWorld(cfg, pack_scenes_ex(scenes), fleet=pack_fleet(scenes), K=7, types=types, robot_type=pack_robot_types(scenes))
    bodies = [body for b in range(4) for body in o.bodies(b)]
    assert sorted({len(p) for p in bodies}) == [3, 4]
    got = o.robot_clearances(bodies)
    want = [min(clearance_robots(bodies[n], bodies[b * 7 + j]) for j in range(7) if b * 7 + j != n) for b in range(4) for n in range(b * 7, b * 7 + 7)]
    assert np.array_equal(got, np.array(want))


def test_mixed_swap_is_circle_swap_with_types_and_starts_apart(lib):
    a, b = mixed_swap(16, seed=3, circles=2), mixed_swap(16, seed=3, circles=2)
    assert np.array_equal(pack_fleet(a), pack_fleet(b)) and np.array_equal(pack_robot_types(a), pack_robot_types(b))
    plain = circle_swap(16, robots=6, seed=3, circles=2)
    assert np.array_equal(pack_fleet(a), pack_fleet(plain))  # the builders do not drift
    assert all(np.array_equal(x, y) for x, y in zip(pack_scenes_ex(a), pack_scenes_ex(plain)))
    assert pack_robot_types(a).tolist() == [0, 1, 2, 0, 1, 2] * 16
    assert pack_robot_types(mixed_swap(2, types=(1,), robots=3)).tolist() == [1] * 6
    assert np.array_equal(pack_fleet(mixed_swap(16, seed=3, circles=2)[9:]), pack_fleet(a[9:]))  # seeded per environment
    with pytest.raises(ValueError, match="types"):
        mixed_swap(2, types=(0, 4))
    diff, car, omni = _robots(DIFF, ACKER, OMNI)
    cfg = make_config(diff, LIDAR, 0.1, max_envs=128)
    types = _types([car, omni])
    sc = mixed_swap(128, robots=6, seed=2024)
    assert _check_ex(lib, cfg, types, 128, 6, pack_fleet(sc), pack_robot_types(sc)) == _lib.NB_OK
    # the bodies, each of its own type, are more than 3 m apart at the start
    verts = [np.asarray(r.vertices, np.float64).T for r in (diff, car, omni)]
    for s in sc[:32]:
        bodies = [ow.robot_polygon(r["start"], verts[r["type"]]) for r in s["robots"]]
        assert min(clearance_robots(bodies[i], bodies[j]) for i in range(6) for j in range(i + 1, 6)) > 3.0
    # 8 cars facing the centre of a 5 m circle reach 3.8 m inwards, where they meet: the host check refuses; diff robots fit
    cars = mixed_swap(4, types=(1,), robots=8, radius=5.0, seed=1)
    assert _check_ex(lib, cfg, types, 4, 8, pack_fleet(cars), pack_robot_types(cars)) == _lib.NB_ERR_INVALID
    assert _check_ex(lib, cfg, types, 4, 8, pack_fleet(cars), np.zeros(32, np.int32)) == _lib.NB_OK


def test_mixed_oracle_with_every_robot_type_zero_is_the_oracle():
    """MixedOracleWorld restates only the per-robot parts of OracleWorld: with every robot of type 0 (and other types present in
    the table) scans, reactive choices and steps are OracleWorld's bit for bit."""
    diff, car, omni = _robots(DIFF, ACKER, OMNI)
    scenes = circle_swap(3, robots=4, radius=6.0, seed=2, circles=3)
    for sc in scenes:
        sc["obstacles"] = [dict(ob, behavior=dict(name="rvo", vxmax=0.5, vymax=0.5, wander=True)) for ob in sc["obstacles"]]
    from neupan_b200.world import pack_behaviors
    cfg = dict(kinematics="diff", step_time=0.1, wheelbase=None, angle_min=-math.pi, angle_max=math.pi, range_max=8.0, number=24,
               scan_offset=(0.1, 0.0, 0.0), robot_vertices=np.asarray(diff.vertices, np.float64).T)
    types = [dict(kinematics=r.kinematics, wheelbase=r.L, robot_vertices=np.asarray(r.vertices, np.float64).T) for r in (car, omni)]
    args = (cfg, pack_scenes_ex(scenes), pack_behaviors(scenes), 4)
    a = ow.OracleWorld(*args, fleet=pack_fleet(scenes), K=4)
    b = MixedOracleWorld(*args, fleet=pack_fleet(scenes), K=4, types=types, robot_type=np.zeros(12, np.int32))
    rng = np.random.default_rng(1)
    for _ in range(15):
        assert all(np.array_equal(x, y) for x, y in zip(a.scan(), b.scan()))
        act = np.column_stack([rng.uniform(0.0, 2.0, 12), rng.uniform(-0.5, 0.5, 12)])
        assert all(np.array_equal(x, y) for x, y in zip(a.step(act), b.step(act)))
        assert np.array_equal(a.obs, b.obs) and np.array_equal(a.states, b.states) and np.array_equal(a.goal, b.goal)
        assert np.array_equal(a.robot_clear, b.robot_clear) and np.array_equal(a.fvel, b.fvel)
