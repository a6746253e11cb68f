"""Several robots per environment in the batched world, on the CPU: host validation through nb_world_check_fleet, the packing of
``robots`` scenes, the circle_swap builder and the sanity of tests/world_fleet_oracle.py (no device needed)."""
import ctypes as C
import math

import numpy as np
import pytest

from neupan_b200 import _lib, build as nb_build
from neupan_b200.robot import robot as Robot
from neupan_b200.world import circle_swap, fleet_size, make_config, pack_fleet, pack_scenes_ex, rectangle, scene_paths
from oracle import world as ow
from world_fleet_oracle import OracleWorld, clearance_robot_pairs, clearance_robots

LIDAR = dict(angle_min=-math.pi, angle_max=math.pi, range_min=0.0, range_max=10.0, number=36)
C4_ROBOT = dict(kinematics="diff", length=1.6, width=2.0)


@pytest.fixture(scope="module")
def lib():
    nb_build.build()
    return _lib.load()


def _check(lib, cfg, B, K, rows):
    rows = np.ascontiguousarray(np.asarray(rows, np.float64).reshape(-1, 6))
    return lib.nb_world_check_fleet(C.byref(cfg), B, K, C.c_void_p(rows.ctypes.data))


def test_host_validation_of_fleets(lib):
    rb = Robot(10, 0.1, **C4_ROBOT)
    cfg = make_config(rb, LIDAR, 0.1, max_envs=4)
    ok = [[0.0, 0.0, 0.0, 5.0, 0.0, 0.3], [0.0, 3.0, 0.0, 5.0, 3.0, 0.3]]  # 1.0 m between the 2.0 m wide bodies
    assert _check(lib, cfg, 1, 2, ok) == _lib.NB_OK
    assert _check(lib, cfg, 2, 2, ok + ok) == _lib.NB_OK
    assert _check(lib, cfg, 1, 1, ok[:1]) == _lib.NB_OK
    assert _check(lib, cfg, 1, 16, [[4.0 * k, 0.0, 0.0, 0.0, 0.0, 0.0] for k in range(16)]) == _lib.NB_OK

    def refused(B, K, rows, msg):
        assert _check(lib, cfg, B, K, rows) == _lib.NB_ERR_INVALID
        assert msg in lib.nb_last_error().decode(), lib.nb_last_error().decode()

    refused(1, 0, ok, "K = 0 robots per environment (1..16)")
    refused(1, 17, [[4.0 * k, 0.0, 0.0, 0.0, 0.0, 0.3] for k in range(17)], "K = 17 robots per environment (1..16)")
    refused(5, 1, ok * 3, "B = 5 outside [1, max_envs = 4]")
    for col in range(6):
        for bad in (math.nan, math.inf):
            rows = [list(r) for r in ok + ok]
            rows[3][col] = bad
            refused(2, 2, rows, "environment 1, robot 1: non-finite value")
    refused(2, 2, ok + [ok[0], [0.0, 3.0, 0.0, 5.0, 3.0, -0.1]], "environment 1, robot 1: goal_threshold must be >= 0")
    refused(2, 2, ok + [ok[0], [0.5, 1.5, 0.3, 5.0, 3.0, 0.3]], "environment 1: the start bodies of robots 0 and 1 overlap")
    refused(1, 2, [ok[0], [0.0, 2.0, 0.0, 5.0, 3.0, 0.3]], "environment 0: the start bodies of robots 0 and 1 overlap")  # touching
    refused(1, 3, ok + [[0.0, 0.0, 1.0, 1.0, 1.0, 0.0]], "environment 0: the start bodies of robots 0 and 2 overlap")
    assert lib.nb_world_check_fleet(C.byref(cfg), 1, 2, None) == _lib.NB_ERR_INVALID


def _fleet_scene(robots, obstacles=()):
    return dict(obstacles=list(obstacles), bounds=(-20.0, -20.0, 20.0, 20.0),
                robots=[dict(start=s, goal=g, goal_threshold=t, path=np.array([[s[0], s[1], s[2], 1.0]])) for s, g, t in robots])


def test_packing_of_robots_scenes():
    a = _fleet_scene([((0.0, 0.0, 0.1), (5.0, 0.0), 0.3), ((0.0, 4.0, 0.2), (5.0, 4.0), 0.4)], [dict(center=(9.0, 9.0), radius=1.0)])
    b = _fleet_scene([((1.0, 0.0, 0.5), (6.0, 0.0), 0.2), ((1.0, 4.0, 0.6), (6.0, 4.0), 0.1)])
    assert fleet_size([a, b]) == 2
    rows = pack_fleet([a, b])
    assert rows.shape == (4, 6) and rows.dtype == np.float64 and rows.flags.c_contiguous
    assert rows.tolist() == [[0.0, 0.0, 0.1, 5.0, 0.0, 0.3], [0.0, 4.0, 0.2, 5.0, 4.0, 0.4], [1.0, 0.0, 0.5, 6.0, 0.0, 0.2],
                             [1.0, 4.0, 0.6, 6.0, 4.0, 0.1]]
    obs_begin, obs, _, _, envs, _ = pack_scenes_ex([a, b])
    assert obs_begin.tolist() == [0, 1, 1] and obs.shape == (1, 5)
    assert envs[:, 4:].tolist() == [rows[0].tolist(), rows[2].tolist()]  # the env row carries the first robot
    assert [p[0, 0] for p in scene_paths([a, b])] == [0.0, 0.0, 1.0, 1.0]
    single = dict(obstacles=[], bounds=(-1.0, -1.0, 1.0, 1.0), start=(0.0, 0.0, 0.0), goal=(1.0, 0.0), goal_threshold=0.5, path=None)
    assert fleet_size([single]) == 1 and pack_fleet([single]).tolist() == [[0.0, 0.0, 0.0, 1.0, 0.0, 0.5]]
    with pytest.raises(ValueError, match="same number of robots"):
        fleet_size([a, single])
    with pytest.raises(ValueError, match="1..16"):
        fleet_size([_fleet_scene([((3.0 * k, 0.0, 0.0), (0.0, 0.0), 0.3) for k in range(17)])])


def test_circle_swap_is_seeded_per_environment_and_starts_apart(lib):
    a, b = circle_swap(8, robots=16, seed=3, circles=3), circle_swap(8, robots=16, seed=3, circles=3)
    sub = circle_swap(8, robots=16, seed=3, circles=3)[5:]
    assert all(np.array_equal(pack_fleet([x]), pack_fleet([y])) for x, y in zip(a, b))
    assert np.array_equal(pack_fleet(a[5:]), pack_fleet(sub)) and np.array_equal(pack_scenes_ex(a[5:])[1], pack_scenes_ex(sub)[1])
    assert not np.array_equal(pack_fleet(a[:1]), pack_fleet(a[1:2]))  # a different rotation per environment
    rows = pack_fleet(a)
    assert np.allclose(np.hypot(rows[:, 3], rows[:, 4]), 10.0) and (rows[:, 5] == 0.3).all()
    # each robot faces its goal, the antipode of its slot, within the jitter
    ang = np.arctan2(rows[:, 4] - rows[:, 1], rows[:, 3] - rows[:, 0])
    assert np.abs(np.angle(np.exp(1j * (rows[:, 2] - ang)))).max() <= 0.05 + 1e-12
    assert len(scene_paths(a)) == 8 * 16 and all(len(sc["obstacles"]) == 3 for sc in a)
    rb = Robot(10, 0.1, **C4_ROBOT)
    cfg = make_config(rb, LIDAR, 0.1, max_envs=64)
    for K in (2, 8, 16):
        sc = circle_swap(64, robots=K, seed=11)
        assert _check(lib, cfg, 64, K, pack_fleet(sc)) == _lib.NB_OK
    # the start bodies are well apart at K = 16: more than 1 m between any two
    rv = np.asarray(rb.vertices, np.float64).T
    for sc in a:
        bodies = np.array([ow.robot_polygon(r["start"], rv) for r in sc["robots"]])
        ii, jj = np.nonzero(~np.eye(16, dtype=bool))
        assert clearance_robot_pairs(bodies[ii], bodies[jj]).min() > 1.0


def test_oracle_robot_clearance_is_symmetric_and_vectorised_exactly():
    rng = np.random.default_rng(0)
    rv = np.asarray(Robot(10, 0.1, **C4_ROBOT).vertices, np.float64).T
    P, Q = [], []
    for _ in range(3000):
        s = (rng.uniform(-1, 1), rng.uniform(-1, 1), rng.uniform(-math.pi, math.pi))
        d = rng.uniform(0.0, 4.0)
        a = rng.uniform(-math.pi, math.pi)
        t = (s[0] + d * math.cos(a), s[1] + d * math.sin(a), rng.uniform(-math.pi, math.pi))
        P.append(ow.robot_polygon(s, rv))
        Q.append(ow.robot_polygon(t, rv))
    scalar_pq = np.array([clearance_robots(p, q) for p, q in zip(P, Q)])
    scalar_qp = np.array([clearance_robots(q, p) for p, q in zip(P, Q)])
    assert np.array_equal(scalar_pq, scalar_qp)  # bit for bit
    P, Q = np.asarray(P), np.asarray(Q)
    assert np.array_equal(clearance_robot_pairs(P, Q), scalar_pq) and np.array_equal(clearance_robot_pairs(Q, P), scalar_pq)
    assert (scalar_pq == 0.0).sum() > 100 and (scalar_pq > 0.0).sum() > 1000
    # a square against a turned copy of itself at a known distance
    sq = [tuple(v) for v in rectangle(2.0, 2.0)]
    other = [(x + 3.5, y) for x, y in sq]
    assert clearance_robots(sq, other) == clearance_robots(other, sq) == 1.5


def test_oracle_fleet_of_one_is_the_single_robot_oracle():
    """The fleet oracle at K = 1 from the env rows steps and scans exactly like the parent oracles."""
    from world_rvo_oracle import OracleWorld as RvoOracle
    rb = Robot(10, 0.1, **C4_ROBOT)
    cfg = dict(kinematics="diff", step_time=0.1, wheelbase=rb.L, angle_min=LIDAR["angle_min"], angle_max=LIDAR["angle_max"],
               range_max=LIDAR["range_max"], number=LIDAR["number"], scan_offset=(0.1, 0.0, 0.0), robot_vertices=np.asarray(rb.vertices).T)
    rng = np.random.default_rng(4)
    scenes = [dict(obstacles=[dict(center=tuple(rng.uniform(-5, 5, 2)), radius=0.5, velocity=(0.3, -0.2)),
                              dict(center=tuple(rng.uniform(-5, 5, 2)), vertices=rectangle(1.0, 0.5), velocity=(-0.2, 0.1))],
                   bounds=(-6.0, -6.0, 6.0, 6.0), start=(0.0, 0.0, 0.3), goal=(4.0, 1.0), goal_threshold=0.3) for _ in range(3)]
    packed = pack_scenes_ex(scenes)
    a, b = OracleWorld(cfg, packed), RvoOracle(cfg, packed)
    for _ in range(20):
        act = np.column_stack([rng.uniform(0, 1.5, 3), rng.uniform(-0.5, 0.5, 3)]).astype(np.float32)
        ra, rb_ = a.scan(), b.scan()
        assert all(np.array_equal(x, y) for x, y in zip(ra, rb_))
        sa, sb = a.step(act), b.step(act)
        assert all(np.array_equal(x, y) for x, y in zip(sa, sb))
        assert np.array_equal(a.states, b.states) and np.array_equal(a.obs, b.obs)
