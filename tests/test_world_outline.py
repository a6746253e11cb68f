"""Outline obstacles (any simple polygon, kind 1) in the batched world, on the CPU: the outline clearance on hand-built cases,
its agreement with the convex clearance, host validation through nb_world_check_scenes_ex, oracle scans into notches and onto
outline boundaries, and the non_obs / dyna_non_obs scene builders (no device needed)."""
import ctypes as C
import math

import numpy as np
import pytest

from neupan_b200 import _lib, build as nb_build
from neupan_b200.robot import robot as Robot
from neupan_b200.world import dyna_non_obs, make_config, non_obs, pack_scenes, pack_scenes_ex, random_outline
from oracle import scan as oscan, world as ow
from oracle.world import OracleWorld, clearance_outline, inside_outline

LIDAR = dict(angle_min=-math.pi, angle_max=math.pi, range_min=0.0, range_max=10.0, number=360)
# a U open upwards: the notch is (-1, 1) x (-1, 3), the arms and the base are 2 m thick
U = [(-3.0, -3.0), (3.0, -3.0), (3.0, 3.0), (1.0, 3.0), (1.0, -1.0), (-1.0, -1.0), (-1.0, 3.0), (-3.0, 3.0)]


@pytest.fixture(scope="module")
def lib():
    nb_build.build()
    return _lib.load()


def _square(cx, cy, h=0.5):
    return [(cx - h, cy - h), (cx + h, cy - h), (cx + h, cy + h), (cx - h, cy + h)]


def _scene(obstacles, start=(0.0, 0.0, 0.0), bounds=(-50.0, -50.0, 50.0, 50.0), goal=(100.0, 100.0), thr=0.1):
    return dict(obstacles=obstacles, bounds=bounds, start=start, goal=goal, goal_threshold=thr)


def _cfg(lidar=LIDAR, kin="diff", **kw):
    kw = kw or dict(length=1.6, width=2.0)
    rb = Robot(10, 0.1, kinematics=kin, **kw)
    return dict(kinematics=kin, step_time=0.1, wheelbase=rb.L, angle_min=lidar["angle_min"], angle_max=lidar["angle_max"],
                range_max=lidar["range_max"], number=lidar["number"], scan_offset=lidar.get("scan_offset", (0.0, 0.0, 0.0)),
                robot_vertices=np.asarray(rb.vertices, np.float64).T), rb


def test_robot_in_the_notch_of_a_u_is_clear_where_the_convex_hull_overlaps():
    robot = _square(0.0, 1.0)  # [-0.5, 0.5] x [0.5, 1.5]: 0.5 from both inner walls and from the notch's floor
    assert clearance_outline(robot, U) == 0.5
    hull = [(-3.0, -3.0), (3.0, -3.0), (3.0, 3.0), (-3.0, 3.0)]
    assert ow.clearance_polygon(robot, hull) == 0.0
    assert clearance_outline(_square(0.0, 2.0), U) == 0.5  # higher up the notch: the floor is farther, the walls are not


def test_outline_overlaps_give_zero():
    assert clearance_outline(_square(1.0, 1.0), U) == 0.0            # straddles the notch's right wall
    assert clearance_outline(_square(2.0, 1.0), U) == 0.0            # wholly inside the right arm: no edge meets
    small = [(0.1 * x + 20.0, 0.1 * y) for x, y in U]
    assert clearance_outline(_square(20.0, 0.0, 2.0), small) == 0.0  # the outline wholly inside the robot
    assert clearance_outline(_square(3.5, 0.0), U) == 0.0            # touching the outer right edge x = 3
    assert clearance_outline(_square(2.0, 3.5), U) == 0.0            # lying on the right arm's top: collinear edges overlap
    assert clearance_outline(_square(2.0, 3.75), U) == 0.25
    assert clearance_outline(_square(0.0, 3.5), U) == 0.5            # above the notch's mouth: 0.5 from the arms' inner corners


def test_vertex_to_vertex_diagonal():
    robot = [(4.0, 4.0), (5.0, 4.0), (5.0, 5.0), (4.0, 5.0)]
    assert clearance_outline(robot, U) == math.sqrt(2.0)


def test_even_odd_inside_of_a_u():
    assert not inside_outline(U, 0.0, 1.0) and inside_outline(U, 2.0, 1.0) and inside_outline(U, 0.0, -2.0) and not inside_outline(U, 5.0, 0.0)


def _convex(rng, c):
    n = int(rng.integers(3, 9))
    ang = np.sort(rng.uniform(0, 2 * np.pi - 0.01, n)) + np.arange(n) * 1e-3
    r = rng.uniform(0.3, 1.5)
    return [(c[0] + r * math.cos(a), c[1] + r * math.sin(a)) for a in ang]


def test_convex_polygons_given_as_outlines_match_clearance_polygon():
    rng = np.random.default_rng(3)
    separated = overlapping = 0
    for _ in range(3000):
        poly = _convex(rng, rng.uniform(-3, 3, 2))
        robot = ow.robot_polygon(rng.uniform(-2, 2, 3), [(-0.8, -1.0), (0.8, -1.0), (0.8, 1.0), (-0.8, 1.0)])
        a, b = ow.clearance_polygon(robot, poly), clearance_outline(robot, poly)
        if a > 0.0:
            separated += 1
            assert a == b  # the same distance loops in the same order: bit for bit
            assert clearance_outline(robot, poly[::-1]) > 0.0
        else:
            overlapping += 1
            assert b == 0.0 and clearance_outline(robot, poly[::-1]) == 0.0  # either orientation
    assert separated > 500 and overlapping > 500


# ---- host validation ---------------------------------------------------------------------------------------------------------

def _star(n=16, r_out=1.0, r_in=0.4):
    return [[(r_out if k % 2 == 0 else r_in) * math.cos(2 * math.pi * k / n), (r_out if k % 2 == 0 else r_in) * math.sin(2 * math.pi * k / n)]
            for k in range(n)]


def _check(lib, cfg, packed):
    return lib.nb_world_check_scenes_ex(C.byref(cfg), len(packed[0]) - 1, *[C.c_void_p(a.ctypes.data) for a in packed])


def test_host_validation_of_outlines(lib):
    rb = Robot(10, 0.1, kinematics="diff", length=1.6, width=2.0)
    cfg = make_config(rb, LIDAR, 0.1, max_envs=4)
    ok = lambda outlines, extra=(): _check(lib, cfg, pack_scenes_ex([_scene([dict(center=(20.0, 0.0), outline=o) for o in outlines] + list(extra))]))
    assert ok([_star()]) == _lib.NB_OK
    assert ok([U]) == _lib.NB_OK and ok([U[::-1]]) == _lib.NB_OK
    assert ok([_star()] * 128) == _lib.NB_OK  # 2048 edges
    refusals = [
        ([_star(18)[:17]], "3..16 vertices (got 17)"),
        ([[[0, 0], [2, 2], [2, 0], [0, 1]]], "not simple"),                 # bow-tie
        ([[[0, 0], [1, 0], [1, 0], [0, 1]]], "zero-length edge"),           # repeated vertex
        ([[[0, 0], [1, 0], [2, 0], [3, 0]]], "zero area"),                   # collinear points
        ([[[0, 0], [2, 0], [1, 0], [1, 1]]], "not simple"),                  # a spike folded back onto an edge
        ([[[0, 0], [2, 0], [2, 2], [1, 0.0], [0, 2]]], "not simple"),        # a vertex touching a non-adjacent edge
        ([_star()] * 127 + [_star(14)], None),                               # with the triangle below: 2049 edges
    ]
    for outlines, text in refusals[:-1]:
        assert ok(outlines) == _lib.NB_ERR_INVALID, outlines
        assert text in lib.nb_last_error().decode(), lib.nb_last_error().decode()
    assert ok(refusals[-1][0], [dict(center=(0.0, 5.0), vertices=[[0, 0], [1, 0], [0, 1]])]) == _lib.NB_ERR_INVALID
    assert "2049 polygon edges (at most 2048)" in lib.nb_last_error().decode()
    assert ok([[[0, 0], [1, 0], [0, math.nan]]]) == _lib.NB_ERR_INVALID


def test_ex_entry_point_keeps_the_convex_rules_and_messages(lib):
    rb = Robot(10, 0.1, kinematics="diff", length=1.6, width=2.0)
    cfg = make_config(rb, LIDAR, 0.1, max_envs=4)
    cases = [dict(center=(5.0, 0.0), vertices=[[math.cos(a), math.sin(a)] for a in np.linspace(0, 6, 9)]),  # 9 vertices
             dict(center=(5.0, 0.0), vertices=U),                                                         # not convex
             dict(center=(5.0, 0.0), radius=-1.0)]
    for ob in cases:
        packed = pack_scenes_ex([_scene([ob])])
        assert lib.nb_world_check_scenes(C.byref(cfg), 1, *[C.c_void_p(a.ctypes.data) for a in packed[:5]]) == _lib.NB_ERR_INVALID
        old = lib.nb_last_error().decode()
        assert _check(lib, cfg, packed) == _lib.NB_ERR_INVALID and lib.nb_last_error().decode() == old
        assert lib.nb_world_check_scenes_ex(C.byref(cfg), 1, *[C.c_void_p(a.ctypes.data) for a in packed[:5]], None) == _lib.NB_ERR_INVALID
        assert lib.nb_last_error().decode() == old
    packed = pack_scenes_ex([_scene([dict(center=(5.0, 0.0), outline=U)])])
    packed[5][0] = 2
    assert _check(lib, cfg, packed) == _lib.NB_ERR_INVALID and "kind 2" in lib.nb_last_error().decode()
    packed[5][0] = 0  # the same vertices as a convex polygon: refused as today
    assert _check(lib, cfg, packed) == _lib.NB_ERR_INVALID and "not a convex polygon" in lib.nb_last_error().decode()


def test_pack_scenes_is_unchanged_without_outlines_and_refuses_outlines():
    scenes = [_scene([dict(center=(1.0, 2.0), radius=0.5, velocity=(0.1, 0.2)), dict(center=(3.0, 4.0), vertices=[[0, 0], [1, 0], [0, 1]])])]
    five, six = pack_scenes(scenes), pack_scenes_ex(scenes)
    assert len(five) == 5 and all(np.array_equal(a, b) and a.dtype == b.dtype for a, b in zip(five, six[:5]))
    assert six[5].dtype == np.int32 and not six[5].any()
    with pytest.raises(ValueError):
        pack_scenes([_scene([dict(center=(0.0, 0.0), outline=U)])])
    with pytest.raises(ValueError):
        pack_scenes_ex([_scene([dict(center=(0.0, 0.0), outline=U, vertices=U)])])


# ---- scans -------------------------------------------------------------------------------------------------------------------

def test_a_beam_into_a_notch_reaches_its_inner_wall():
    # the U turned to open towards the sensor: the notch is (7, 11) x (-1, 1) in the world, its inner wall at x = 11
    u_left = [(-y, x) for x, y in U]
    lidar = dict(angle_min=0.0, angle_max=0.0, range_min=0.0, range_max=20.0, number=1)
    cfg, _ = _cfg(lidar)
    w = OracleWorld(cfg, pack_scenes_ex([_scene([dict(center=(10.0, 0.0), outline=u_left)])]))
    r, _, hit, _, _ = w.scan()
    assert r[0, 0] == 11.0 and hit[0, 0] == 0
    hull = OracleWorld(cfg, pack_scenes([_scene([dict(center=(10.0, 0.0), vertices=[(-3, -3), (3, -3), (3, 3), (-3, 3)])])]))
    assert hull.scan()[0][0, 0] == 7.0


def _boundary_distance(p, scene):
    d = math.inf
    for ob in scene["obstacles"]:
        cx, cy = ob["center"]
        shape = "vertices" if "vertices" in ob else ("outline" if "outline" in ob else None)
        if shape:
            v = np.asarray(ob[shape]) + (cx, cy)
            for k in range(len(v)):
                a, b = v[k], v[(k + 1) % len(v)]
                d = min(d, ow.seg_dist(p[0], p[1], a[0], a[1], b[0], b[1]))
        else:
            d = min(d, abs(math.hypot(p[0] - cx, p[1] - cy) - ob["radius"]))
    return d


@pytest.mark.parametrize("builder", [non_obs, dyna_non_obs])
def test_oracle_scans_of_outline_scenes_map_to_points_on_the_boundaries(builder):
    scenes = builder(4, seed=13)
    rng = np.random.default_rng(1)
    for sc in scenes:  # robots among the obstacles, turned at random
        sc["start"] = (rng.uniform(8, 40), rng.uniform(17, 33), rng.uniform(-np.pi, np.pi))
    offset = (0.2, -0.1, 0.1)
    lidar = dict(LIDAR, number=361, scan_offset=offset)
    cfg, _ = _cfg(lidar)
    w = OracleWorld(cfg, pack_scenes_ex(scenes))
    ranges, _, hit, _, _ = w.scan()
    n = n_outline = 0
    for b, sc in enumerate(scenes):
        pts = oscan.scan_to_point(w.states[b].reshape(3, 1), dict(lidar, ranges=ranges[b]), scan_offset=offset)
        for p in pts.T:
            assert _boundary_distance(p, sc) < 1e-9
            n += 1
        n_outline += sum(1 for h in hit[b] if h >= 0 and "outline" in sc["obstacles"][h])
    assert n > 100 and n_outline > 50


# ---- scene builders ----------------------------------------------------------------------------------------------------------

def _same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if k == "obstacles":
            assert len(a[k]) == len(b[k])
            for x, y in zip(a[k], b[k]):
                assert x.keys() == y.keys() and all(np.array_equal(np.asarray(x[f]), np.asarray(y[f])) for f in x)
        else:
            assert np.array_equal(np.asarray(a[k]), np.asarray(b[k]))


def _min_start_clearance(sc, robot_vertices):
    robot = ow.robot_polygon(sc["start"], robot_vertices)
    best = math.inf
    for ob in sc["obstacles"]:
        cx, cy = ob["center"]
        if "radius" in ob:
            best = min(best, ow.clearance_circle(robot, cx, cy, ob["radius"]))
        else:
            poly = [(cx + x, cy + y) for x, y in np.asarray(ob.get("outline", ob.get("vertices")))]
            best = min(best, clearance_outline(robot, poly))
    return best


@pytest.mark.parametrize("builder, kin", [(dyna_non_obs, "diff"), (non_obs, "acker")])
def test_scene_builders_after_the_examples(lib, builder, kin):
    scenes = builder(64, seed=21)
    for x, y in zip(builder(70, seed=21)[10:64], scenes[10:]):
        _same(x, y)
    assert any(not np.array_equal(np.asarray(scenes[0]["obstacles"][k].get("outline", 0)), np.asarray(scenes[1]["obstacles"][k].get("outline", 0)))
               for k in range(11))
    kw = dict(length=4.6, width=1.6, wheelbase=3) if kin == "acker" else dict(length=1.6, width=2.0)
    cfg, rb = _cfg(kin=kin, **kw)
    assert _check(lib, make_config(rb, LIDAR, 0.1, max_envs=64), pack_scenes_ex(scenes)) == _lib.NB_OK  # every outline simple
    shapes = {}
    for sc in scenes:
        assert len(sc["obstacles"]) == 11 and sc["start"] == (-1.0, 25.0, 0.0) and sc["goal"] == (50.0, 25.0)
        assert np.allclose(sc["path"][[0, -1], :2], [[-1.0, 25.0], [50.0, 25.0]])
        assert _min_start_clearance(sc, cfg["robot_vertices"]) > 1.0
        for ob in sc["obstacles"]:
            key = "outline" if "outline" in ob else ("square" if "vertices" in ob else f"r{ob['radius']}")
            shapes[key] = shapes.get(key, 0) + 1
            if "outline" in ob:
                v = np.asarray(ob["outline"])
                r = np.hypot(v[:, 0], v[:, 1])
                assert 4 <= len(v) <= 9 and r.min() >= 0.05 - 1e-12 and r.max() <= (3.0 if builder is dyna_non_obs else 2.0) + 1e-12
    if builder is non_obs:
        assert sc["bounds"] == (-2.0, 5.0, 51.0, 47.0) and sc["goal_threshold"] == 0.3
        assert shapes == {"outline": 64 * 11}
        assert [ob["center"] for ob in sc["obstacles"]][5] == [ob["center"] for ob in sc["obstacles"]][8] == (16.0, 26.0)
        assert all("velocity" not in ob for sc in scenes for ob in sc["obstacles"])
    else:
        assert sc["bounds"] == (5.0, 15.0, 45.0, 35.0) and sc["goal_threshold"] == 0.4
        assert set(shapes) == {"outline", "square", "r1.5", "r1.0"} and min(shapes.values()) > 64 * 11 / 4 * 0.7
        for sc in scenes:
            for ob in sc["obstacles"]:
                assert 5.0 <= ob["center"][0] <= 45.0 and 15.0 <= ob["center"][1] <= 35.0
                assert all(-1.0 <= v <= 1.0 for v in ob["velocity"])


def test_random_outline_is_star_shaped_and_simple(lib):
    rng = np.random.default_rng(4)
    outlines = [random_outline(rng, rng.uniform(0.5, 1.5), rng.uniform(0.0, 1.0), rng.uniform(0.0, 1.0), int(rng.integers(3, 17)))
                for _ in range(256)]
    rb = Robot(10, 0.1, kinematics="diff", length=1.6, width=2.0)
    scenes = [_scene([dict(center=(20.0, 0.0), outline=o) for o in outlines[i:i + 64]]) for i in range(0, 256, 64)]
    assert _check(lib, make_config(rb, LIDAR, 0.1, max_envs=4), pack_scenes_ex(scenes)) == _lib.NB_OK
    for o in outlines:
        assert inside_outline([tuple(v) for v in o], 0.0, 0.0)  # the centre sees every vertex: it lies inside
