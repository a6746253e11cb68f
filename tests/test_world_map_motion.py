"""Obstacles in occupancy maps on the CPU (no device needed): the refusals of nb_world_check_map_contact, the move rule by hand
(tests/world_map_motion_oracle.py), the wander goal test against a brute-force check over every occupied cell, the draw numbering
across rejections, an invariant run in which no moving obstacle ever touches the map, and the maze / cave builders."""
import ctypes as C
import hashlib
import math

import numpy as np
import pytest

from neupan_b200 import _lib, build as nb_build
from neupan_b200.robot import robot as Robot
from neupan_b200.world import (cave, make_config, maze, pack_behaviors, pack_map_contact, pack_maps, pack_scenes_ex)
from oracle.world import draw_goal
from world_map_motion_oracle import MapMotionOracleWorld, cell_polygons, footprint_touches_cells, segment_near_cells

LIDAR = dict(angle_min=-math.pi, angle_max=math.pi, range_min=0.0, range_max=10.0, number=8)
DIFF = dict(kinematics="diff", length=1.6, width=2.0)
DT = 0.1


@pytest.fixture(scope="module")
def lib():
    nb_build.build()
    return _lib.load()


def _robot():
    return Robot(10, DT, **DIFF)


def _cfg():
    rb = _robot()
    return dict(kinematics="diff", step_time=DT, wheelbase=rb.L, angle_min=LIDAR["angle_min"], angle_max=LIDAR["angle_max"],
                range_max=LIDAR["range_max"], number=LIDAR["number"], scan_offset=(0.0, 0.0, 0.0),
                robot_vertices=np.asarray(rb.vertices, np.float64).T)


def _scene(occ, obstacles, res=1.0, origin=(0.0, 0.0), bounds=(0.0, 0.0, 20.0, 20.0), block=True, start=(18.5, 18.5, 0.0)):
    return dict(obstacles=obstacles, bounds=bounds, start=start, goal=(18.5, 1.5), goal_threshold=0.3, path=None,
                map=dict(occupancy=occ, origin=origin, resolution=res, blocks_obstacles=block))


def _oracle(scenes, seed=0):
    beh = pack_behaviors(scenes) if any("behavior" in ob for sc in scenes for ob in sc["obstacles"]) else None
    return MapMotionOracleWorld(_cfg(), pack_scenes_ex(scenes), beh, seed, maps=pack_maps(scenes), block=pack_map_contact(scenes))


def _check(lib, scenes, flags=None):
    cfg = make_config(_robot(), LIDAR, DT, max_envs=8)
    packed = pack_scenes_ex(scenes)
    beh = pack_behaviors(scenes) if any("behavior" in ob for sc in scenes for ob in sc["obstacles"]) else None
    maps, bits, env_map = pack_maps(scenes)
    flags = pack_map_contact(scenes) if flags is None else np.asarray(flags, np.int32)
    return lib.nb_world_check_map_contact(C.byref(cfg), len(scenes), *[C.c_void_p(a.ctypes.data) for a in packed],
                                          C.c_void_p(beh.ctypes.data) if beh is not None else None, len(maps), maps,
                                          C.c_void_p(bits.ctypes.data), C.c_void_p(env_map.ctypes.data), C.c_void_p(flags.ctypes.data))


def _walled(n=20):
    occ = np.zeros((n, n), bool)
    occ[0, :] = occ[-1, :] = occ[:, 0] = occ[:, -1] = True
    return occ


# ---- refusals ---------------------------------------------------------------------------------------------------------------

def test_refusals_name_the_environment_and_obstacle(lib):
    occ = _walled()
    ok = [_scene(occ, [dict(center=(5.0, 5.0), radius=0.4, velocity=(0.5, 0.2)), dict(center=(0.5, 0.5), radius=2.0)]),
          {k: v for k, v in _scene(occ, []).items() if k != "map"}]
    assert _check(lib, ok) == _lib.NB_OK  # a static obstacle may overlap a wall

    def refused(rc, msg):
        assert rc == _lib.NB_ERR_INVALID
        assert msg in lib.nb_last_error().decode(), lib.nb_last_error().decode()

    refused(_check(lib, ok, flags=[2, 0]), "environment 0: map contact flag 2 (0 or 1)")
    refused(_check(lib, ok, flags=[-1, 0]), "environment 0: map contact flag -1 (0 or 1)")
    refused(_check(lib, ok, flags=[1, 1]), "environment 1: its map blocks obstacles but it has no map")
    touching = [_scene(occ, [dict(center=(1.3, 5.0), radius=0.4, velocity=(0.5, 0.0))])]
    refused(_check(lib, touching), "environment 0, obstacle 0: moves but its start footprint overlaps or touches occupied cell (0, ")
    square = [[-0.5, -0.5], [0.5, -0.5], [0.5, 0.5], [-0.5, 0.5]]
    refused(_check(lib, [_scene(occ, [dict(center=(1.5, 5.0), vertices=square, velocity=(0.1, 0.0))])]),
            "environment 0, obstacle 0: moves but its start footprint")
    refused(_check(lib, [_scene(occ, [dict(center=(1.5, 5.0), outline=square, velocity=(0.1, 0.0))])]),
            "environment 0, obstacle 0: moves but its start footprint")
    assert _check(lib, [_scene(occ, [dict(center=(1.51, 5.0), vertices=square, velocity=(0.1, 0.0))])]) == _lib.NB_OK
    fast = [_scene(occ, [dict(center=(5.0, 5.0), radius=0.4), dict(center=(9.0, 9.0), radius=0.4, velocity=(8.0, 6.0))])]
    refused(_check(lib, fast), "environment 0, obstacle 1: top speed 10 m/s * step_time = 1 m is not below the map's resolution 1 m")
    rvo = [_scene(occ, [dict(center=(9.0, 9.0), radius=0.4, behavior=dict(name="rvo", vxmax=8.0, vymax=6.0, wander=True))])]
    refused(_check(lib, rvo), "environment 0, obstacle 0: top speed 10 m/s")
    still_rvo = [_scene(occ, [dict(center=(1.2, 9.0), radius=0.4, behavior=dict(name="rvo", vxmax=0.5, vymax=0.5))])]
    refused(_check(lib, still_rvo), "environment 0, obstacle 0: moves but its start footprint")  # reactive counts as moving
    assert _check(lib, [_scene(occ, fast[0]["obstacles"], block=False)]) == _lib.NB_OK  # unblocked: nothing checked


# ---- the move rule ----------------------------------------------------------------------------------------------------------

def _one(occ, ob, res=1.0, bounds=(0.0, 0.0, 20.0, 20.0)):
    o = _oracle([_scene(occ, [ob], res=res, bounds=bounds)])
    o.step(np.zeros((1, 2)))
    return o


def test_move_rule_by_hand():
    occ = _walled()
    occ[:, 10] = True  # a vertical wall x in [10, 11]
    # moving (+x, +y) into the vertical wall: the y move alone (C), x velocity reversed
    o = _one(occ, dict(center=(9.5, 5.0), radius=0.45, velocity=(0.8, 0.5)))
    assert o.taken == dict(B=0, C=1, D=0) and o.bounces[0] == 1
    assert tuple(o.obs[0, :4]) == (9.5, 5.0 + 0.5 * DT, -0.8, 0.5)
    occ = _walled()
    occ[10, :] = True  # a horizontal wall y in [10, 11]
    o = _one(occ, dict(center=(5.0, 9.5), radius=0.45, velocity=(0.5, 0.8)))
    assert o.taken == dict(B=1, C=0, D=0)
    assert tuple(o.obs[0, :4]) == (5.0 + 0.5 * DT, 9.5, 0.5, -0.8)
    occ[:, 10] = True  # and a vertical one: a corner
    o = _one(occ, dict(center=(9.5, 9.5), radius=0.45, velocity=(0.8, 0.8)))
    assert o.taken == dict(B=0, C=0, D=1)
    assert tuple(o.obs[0, :4]) == (9.5, 9.5, -0.8, -0.8)
    # a pocket narrower than one step each way: 0.05 m to every wall, steps of 0.08 m
    occ = np.ones((20, 20), bool)
    occ[5, 5] = False
    o = _one(occ, dict(center=(5.5, 5.5), radius=0.45, velocity=(0.8, 0.8)))
    assert o.taken == dict(B=0, C=0, D=1) and o.bounces[0] == 1
    o.step(np.zeros((1, 2)))
    assert o.taken["D"] == 2 and tuple(o.obs[0, :4]) == (5.5, 5.5, 0.8, 0.8)  # reversed twice
    # the rectangle mirror lands in a wall: x mirrored at xmax = 12, the y move goes into the wall above -> B with both reversed
    occ = _walled()
    occ[10, :] = True
    o = _one(occ, dict(center=(11.95, 9.5), radius=0.45, velocity=(0.8, 0.8)), bounds=(0.0, 0.0, 12.0, 20.0))
    assert o.taken == dict(B=1, C=0, D=0)
    assert tuple(o.obs[0, :4]) == (2.0 * 12.0 - (11.95 + 0.8 * DT), 9.5, -0.8, -0.8)
    # no contact, and static obstacles never move or bounce even inside a wall
    o = _one(_walled(), dict(center=(5.0, 5.0), radius=0.45, velocity=(0.8, 0.5)))
    assert o.bounces[0] == 0 and tuple(o.obs[0, :2]) == (5.0 + 0.8 * DT, 5.0 + 0.5 * DT)
    o = _one(_walled(), dict(center=(0.5, 0.5), radius=0.45))
    assert o.bounces[0] == 0 and tuple(o.obs[0, :4]) == (0.5, 0.5, 0.0, 0.0)


# ---- the goal test ----------------------------------------------------------------------------------------------------------

def _shape_obstacle(rng, kind, c):
    if kind == 0:
        return dict(center=c, radius=float(rng.uniform(0.2, 0.7)))
    ang = np.sort(rng.uniform(0, 2 * np.pi, int(rng.integers(3, 8))))
    r = rng.uniform(0.2, 0.7, len(ang))
    pts = np.stack([r * np.cos(ang), r * np.sin(ang)], 1)
    if kind == 1:
        ang = np.linspace(0, 2 * np.pi, len(ang), endpoint=False) + rng.uniform(0, 1)
        pts = 0.5 * np.stack([np.cos(ang), np.sin(ang)], 1)
        return dict(center=c, vertices=pts)
    return dict(center=c, outline=pts)


def test_goal_test_is_the_brute_force_check_over_every_occupied_cell():
    rng = np.random.default_rng(4)
    agree = {True: 0, False: 0}
    for t in range(120):
        res = float(rng.choice([0.05, 0.2, 0.5, 1.0]))
        n = int(16.0 / res)
        occ = rng.uniform(size=(n, n)) < rng.uniform(0.002, 0.05)
        origin = tuple(rng.uniform(-2.0, 2.0, 2))
        c = tuple(rng.uniform(2.0, 14.0, 2))
        ob = _shape_obstacle(rng, t % 3, c)
        o = _oracle([_scene(occ, [ob], res=res, origin=origin)])
        g = tuple(rng.uniform(0.0, 16.0, 2)) if t % 10 else c
        got = o.goal_clear(0, 0, c[0], c[1], g[0], g[1])
        jj, ii = np.nonzero(occ)
        Q = cell_polygons(o.table, 0, ii, jj)
        touch = footprint_touches_cells(o.shape(0), g[0], g[1], Q).any()
        near = (g != c) and segment_near_cells(c[0], c[1], g[0], g[1], Q, float(o.radius[0])).any()
        assert got == (not touch and not near), t
        agree[got] += 1
    assert agree[True] > 10 and agree[False] > 10


def test_segment_as_a_two_vertex_polygon():
    """The degenerate SAT: a segment past a cell's corner, along its side and through it."""
    Q = np.array([[[0.0, 0.0], [1.0, 0.0], [1.0, 1.0], [0.0, 1.0]]])
    assert not segment_near_cells(-1.0, 2.0, 2.0, 2.0, Q, 0.5).any()   # 1 m above the cell
    assert segment_near_cells(-1.0, 1.4, 2.0, 1.4, Q, 0.5).any()        # 0.4 m above it
    assert segment_near_cells(-1.0, -1.0, 2.0, 2.0, Q, 0.01).any()      # through it
    assert not segment_near_cells(0.9, -0.5, 2.4, 1.0, Q, 0.25).any()   # past the corner (1, 0) at 0.4 / sqrt(2) = 0.283 m
    assert segment_near_cells(0.9, -0.5, 2.4, 1.0, Q, 0.3).any()


def test_draws_use_up_their_numbers_and_sixteen_failures_park():
    occ = np.zeros((20, 20), bool)
    occ[:, 4:] = True  # only x < 4 is free: most draws in the 20 x 20 rectangle are rejected
    beh = dict(name="rvo", vxmax=0.5, vymax=0.5, wander=True)
    o = _oracle([_scene(occ, [dict(center=(2.0, 10.0), radius=0.3, behavior=beh)], start=(1.0, 1.0, 0.0))], seed=3)
    assert tuple(o.goal[0]) == (2.0, 10.0) and o.draws[0] == 0  # goal = centre, draw 0: the first goal is drawn through the test
    o.step(np.zeros((1, 2)))
    n = int(o.draws[0])
    first = next(k for k in range(16) if o.goal_clear(0, 0, 2.0, 10.0, *draw_goal(3, 0, 0, k, (0.0, 0.0, 20.0, 20.0))))
    assert n == first + 1 and o.rejected_draws == first > 0
    assert tuple(o.goal[0]) == draw_goal(3, 0, 0, first, (0.0, 0.0, 20.0, 20.0))
    occ = np.ones((20, 20), bool)
    occ[10, 1] = False  # a one-cell pocket: no goal of these draws has a clear footprint
    o = _oracle([_scene(occ, [dict(center=(1.5, 10.5), radius=0.3, behavior=beh)], start=(1.0, 1.0, 0.0))], seed=3)
    o.step(np.zeros((1, 2)))
    assert o.draws[0] == 16 and tuple(o.goal[0]) == (1.5, 10.5) and tuple(o.obs[0, 2:4]) == (0.0, 0.0)
    o.step(np.zeros((1, 2)))
    assert o.draws[0] == 32 and o.rejected_draws == 32


def test_no_moving_obstacle_ever_touches_the_map():
    """200 oracle steps of four random noise maps with constant and reactive circles, polygons and outlines."""
    rng = np.random.default_rng(8)
    scenes = []
    for b in range(4):
        res = (0.2, 0.5, 0.25, 1.0)[b]
        n = int(20.0 / res)
        occ = rng.uniform(size=(n, n)) < 0.04
        occ[0, :] = occ[-1, :] = occ[:, 0] = occ[:, -1] = True
        obs = []
        for i in range(6):
            c = tuple(rng.uniform(3.0, 17.0, 2))
            ob = _shape_obstacle(rng, i % 3, c)
            top = 0.9 * res / DT
            if i % 2:
                ob["behavior"] = dict(name="rvo", vxmax=top / 1.5, vymax=top / 1.5, wander=True, acce=top / 1.5, grid=top / 8)
            else:
                a = rng.uniform(-math.pi, math.pi)
                ob["velocity"] = (top * math.cos(a), top * math.sin(a))
            cx, cy = (np.arange(n) + 0.5) * res, (np.arange(n) + 0.5) * res
            occ[np.hypot(cx[None, :] - c[0], cy[:, None] - c[1]) <= 0.75 + 1.5 * res] = False
            obs.append(ob)
        scenes.append(_scene(occ, obs, res=res, start=(1.0, 1.0, 0.0)))
    o = _oracle(scenes, seed=2)
    for k in range(200):
        o.step(np.zeros((4, 2)))
        assert not any(o.obstacle_touches_map(q) for q in range(len(o.obs))), k
    assert o.bounces.sum() > 0 and sum(o.taken.values()) == o.bounces.sum()


# ---- builders ---------------------------------------------------------------------------------------------------------------

def _fingerprint(scenes):
    h = hashlib.sha256()
    for sc in scenes:
        h.update(np.ascontiguousarray(sc["map"]["occupancy"]).tobytes()); h.update(np.ascontiguousarray(sc["path"]).tobytes())
        h.update(repr((sc["obstacles"], sc["bounds"], sc["start"], sc["goal"], sc["goal_threshold"], sc["map"]["origin"], sc["map"]["resolution"],
                       sorted(sc["map"]))).encode())
    return h.hexdigest()


def test_builders_without_movers_are_unchanged_and_with_movers_start_clear(lib):
    # the scenes these builders made before they took movers
    assert _fingerprint(maze(3, seed=1)) == "890cfcf93cbd693e13dd46460372232cb36f13ea11c74fbb359a225b2f3bdb76"
    assert _fingerprint(cave(2, seed=2, size=(20.0, 20.0))) == "e40822c7120f0bf859d0fc5a18f41d87157f58194add779fb4cd6a77419d52b8"
    assert _fingerprint(maze(3, seed=1, movers=0)) == _fingerprint(maze(3, seed=1))
    for scenes in (maze(4, seed=1, movers=8), maze(4, seed=1, movers=8, behavior="rvo"), cave(3, seed=2, movers=12),
                   cave(3, seed=2, movers=12, behavior="rvo", resolution=0.1)):
        assert all(sc["map"]["blocks_obstacles"] for sc in scenes)
        assert _check(lib, scenes) == _lib.NB_OK, lib.nb_last_error()
        for sc in scenes:
            sx, sy = sc["start"][:2]
            for ob in sc["obstacles"]:
                assert 0.3 <= ob["radius"] <= 0.6 and math.hypot(*ob["velocity"]) < 0.5
                assert math.hypot(ob["center"][0] - sx, ob["center"][1] - sy) >= 4.0
    assert maze(2, seed=1, movers=3)[1]["obstacles"] != maze(2, seed=1, movers=3)[0]["obstacles"]
