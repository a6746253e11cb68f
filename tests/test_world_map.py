"""Occupancy maps in the batched world, on the CPU: the refusals of nb_world_check_maps, the bit packing of pack_maps, the oracle's
grid walk against a brute-force caster over the boundary faces of the occupied cells, its windowed map clearance against a
brute-force minimum over every occupied cell, and the maze / cave builders (no device needed)."""
import ctypes as C
import math

import numpy as np
import pytest

from neupan_b200 import _lib, build as nb_build
from neupan_b200.robot import robot as Robot
from neupan_b200.world import cave, dyna_obs, make_config, make_robot_type, maze, pack_fleet, pack_maps, pack_robot_types
from oracle import world as ow
from oracle.world import cast, clearance_robot_pairs
from world_map_oracle import MapTable, cell_polygons, map_cast, map_clearance

LIDAR = dict(angle_min=-math.pi, angle_max=math.pi, range_min=0.0, range_max=10.0, number=36)
DIFF = dict(kinematics="diff", length=1.6, width=2.0)
ACKER = dict(kinematics="acker", length=4.6, width=1.6, wheelbase=3)


@pytest.fixture(scope="module")
def lib():
    nb_build.build()
    return _lib.load()


def _scene(occ, origin=(0.0, 0.0), res=1.0, start=(0.5, 0.5, 0.0)):
    return dict(obstacles=[], bounds=(-50.0, -50.0, 50.0, 50.0), start=start, goal=(40.0, 40.0), goal_threshold=0.3, path=None,
                map=dict(occupancy=occ, origin=origin, resolution=res))


def _check(lib, cfg, scenes, window=1.0, robots=True, T=0, types=None, maps=None):
    maps, bits, env_map = maps or pack_maps(scenes)
    rows, rtype = pack_fleet(scenes), pack_robot_types(scenes)
    K = len(rows) // len(scenes)
    return lib.nb_world_check_maps(C.byref(cfg), T, types, len(scenes), K, C.c_void_p(rows.ctypes.data) if robots else None,
                                   C.c_void_p(rtype.ctypes.data), len(maps), maps, C.c_void_p(bits.ctypes.data),
                                   C.c_void_p(env_map.ctypes.data), window)


# ---- refusals ---------------------------------------------------------------------------------------------------------------

def test_refusals_name_the_map_environment_or_robot(lib):
    diff, car = Robot(10, 0.1, **DIFF), Robot(10, 0.1, **ACKER)
    cfg = make_config(diff, LIDAR, 0.1, max_envs=4)
    occ = np.zeros((10, 40), bool)
    occ[0, :] = True  # a wall along y in [0, 1]
    ok = [_scene(occ, start=(5.0, 5.0, 0.0))]
    ok.append({k: v for k, v in ok[0].items() if k != "map"})  # environment 1 has no map
    assert _check(lib, cfg, ok) == _lib.NB_OK

    def refused(rc, msg):
        assert rc == _lib.NB_ERR_INVALID
        assert msg in lib.nb_last_error().decode(), lib.nb_last_error().decode()

    def with_map(**fields):
        maps, bits, env_map = pack_maps(ok)
        for k, v in fields.items():
            if k == "origin":
                maps[0].origin = (C.c_double * 2)(*v)
            else:
                setattr(maps[0], k, v)
        return maps, bits, env_map

    refused(_check(lib, cfg, ok, maps=with_map(width=0)), "map 0: width 0 and height 10 must be in 1..8192")
    refused(_check(lib, cfg, ok, maps=with_map(height=8193)), "map 0: width 40 and height 8193 must be in 1..8192")
    refused(_check(lib, cfg, ok, maps=with_map(origin=(math.nan, 0.0))), "map 0: the origin is not finite")
    refused(_check(lib, cfg, ok, maps=with_map(origin=(0.0, math.inf))), "map 0: the origin is not finite")
    for res in (0.0099, 0.0, -1.0, math.nan, math.inf):
        refused(_check(lib, cfg, ok, maps=with_map(resolution=res)), "map 0: the resolution must be finite and >= 0.01 m")
    assert _check(lib, cfg, ok, maps=with_map(resolution=0.01, origin=(0.0, -5.0))) == _lib.NB_OK  # the limit
    maps, bits, env_map = pack_maps(ok)
    bits[2 * 3 + 1] |= np.uint32(1 << 8)  # row 3, word 1: cell 40 is past width 40
    refused(_check(lib, cfg, ok, maps=(maps, bits, env_map)), "map 0: row 3 has padding bits set past width 40")
    for e in (-2, 1):
        refused(_check(lib, cfg, ok, maps=(maps, pack_maps(ok)[1], np.array([0, e], np.int32))), f"environment 1: map {e} outside -1..0")
    for win in (0.0, -1.0, 10.5, math.nan, math.inf):
        refused(_check(lib, cfg, ok, window=win), "outside (0, 10] m")
    assert _check(lib, cfg, ok, window=10.0) == _lib.NB_OK
    # P: the count of maps
    maps, bits, env_map = pack_maps(ok)
    for P in (0, 5):
        rows = pack_fleet(ok)
        rc = lib.nb_world_check_maps(C.byref(cfg), 0, None, 2, 1, C.c_void_p(rows.ctypes.data), None, P, maps, C.c_void_p(bits.ctypes.data),
                                     C.c_void_p(env_map.ctypes.data), 1.0)
        refused(rc, f"P = {P} maps outside [1, max_envs = 4]")
    rc = lib.nb_world_check_maps(C.byref(cfg), 0, None, 2, 1, None, None, 1, None, C.c_void_p(bits.ctypes.data), C.c_void_p(env_map.ctypes.data), 1.0)
    refused(rc, "nb_world maps: null argument")
    # start bodies: C4's 1.6 x 2.0 body at (5, 2) reaches y = 1.2 > 1 clear; at y = 1.8 it overlaps the wall; at y = 2.0 its lower
    # edge lies on the wall's face y = 1 (touching counts)
    for y, good in ((2.2, True), (1.8, False), (2.0, False)):
        sc = [_scene(occ, start=(5.0, y, 0.0))]
        rc = _check(lib, cfg, sc)
        if good:
            assert rc == _lib.NB_OK
        else:
            refused(rc, "environment 0, robot 0: the start body overlaps or touches occupied cell (")
        assert _check(lib, cfg, sc, robots=False) == _lib.NB_OK  # without robots: the maps alone
    # each robot its own polygon: the car (rear axle at its state, 3.8 m ahead) reaches an occupied column at x = 9 from x = 5.5
    col = np.zeros((10, 40), bool)
    col[:, 9] = True
    fleet = [dict(_scene(col), robots=[dict(start=(2.0, 5.0, 0.0), goal=(1.0, 1.0), goal_threshold=0.3, path=None),
                                       dict(start=(5.5, 2.0, 0.0), goal=(1.0, 1.0), goal_threshold=0.3, path=None, type=1)])]
    types = (_lib.WorldRobotType * 1)(make_robot_type(car))
    refused(_check(lib, cfg, fleet, T=1, types=types), "environment 0, robot 1: the start body overlaps or touches occupied cell (9, ")
    fleet[0]["robots"][1]["type"] = 0  # a diff robot there reaches x = 6.3 only
    assert _check(lib, cfg, fleet, T=1, types=types) == _lib.NB_OK
    # the fleet's own checks come first
    fleet[0]["robots"][1]["start"] = (2.5, 5.0, 0.0)
    refused(_check(lib, cfg, fleet, T=1, types=types), "the start bodies of robots 0 and 1 overlap")


# ---- packing ----------------------------------------------------------------------------------------------------------------

def test_packing_layout_sharing_and_env_map():
    rng = np.random.default_rng(0)
    a = rng.uniform(size=(5, 70)) < 0.3  # 3 words per row, 26 padding bits in the last
    b = rng.uniform(size=(3, 32)) < 0.5  # exactly one word per row
    plain = dyna_obs(1)[0]
    scenes = [_scene(a), _scene(b, origin=(1.0, 2.0), res=0.5), _scene(a), plain, _scene(a, res=0.5)]
    maps, bits, env_map = pack_maps(scenes)
    assert env_map.dtype == np.int32 and env_map.tolist() == [0, 1, 0, -1, 2]  # a shared map is stored once; other origin or res: new
    assert len(maps) == 3 and bits.dtype == np.uint32 and bits.shape == (5 * 3 + 3 * 1 + 5 * 3,)
    assert (maps[1].width, maps[1].height, tuple(maps[1].origin), maps[1].resolution) == (32, 3, (1.0, 2.0), 0.5)
    words = bits[:15].reshape(5, 3)
    for j in range(5):  # row j is y index j; bit i mod 32 of word i / 32 is cell (i, j)
        for i in range(70):
            assert bool((int(words[j, i // 32]) >> (i % 32)) & 1) == a[j, i]
        assert int(words[j, 2]) >> 6 == 0  # padding
    assert MapTable(maps, bits, env_map).occ[1].tolist() == b.tolist()  # the oracle reads back what was packed
    assert pack_maps([plain, plain])[2].tolist() == [-1, -1]


# ---- the grid walk against brute force --------------------------------------------------------------------------------------

def _faces(occ, x0, y0, r):
    """Every boundary face of the occupied cells (a side whose neighbour is free or outside) as cast's edge rows."""
    H, W = occ.shape
    pad = np.pad(occ, 1)
    rows = []
    for j, i in zip(*np.nonzero(occ)):
        X0, X1 = x0 + float(i) * r, x0 + float(i + 1) * r
        Y0, Y1 = y0 + float(j) * r, y0 + float(j + 1) * r
        if not pad[j + 1, i]:
            rows.append((X0, Y0, X0, Y1, 0))
        if not pad[j + 1, i + 2]:
            rows.append((X1, Y0, X1, Y1, 0))
        if not pad[j, i + 1]:
            rows.append((X0, Y0, X1, Y0, 0))
        if not pad[j + 2, i + 1]:
            rows.append((X0, Y1, X1, Y1, 0))
    return np.array(rows, np.float64).reshape(-1, 5)


def _near_corner(x0, y0, r, W, H, sx, sy, dx, dy, tmax, tol=1e-12):
    """Does the ray pass within tol of a grid corner before tmax (+ a cell)?"""
    cx = x0 + np.arange(W + 1) * r
    cy = y0 + np.arange(H + 1) * r
    px, py = np.meshgrid(cx - sx, cy - sy)
    t = px * dx + py * dy
    d = np.abs(px * dy - py * dx)
    return bool(((d < tol * max(1.0, abs(sx), abs(sy), r * max(W, H))) & (t > -r) & (t < tmax + r)).any())


def _table(occ, x0, y0, r):
    return MapTable(*pack_maps([_scene(occ, origin=(x0, y0), res=r)]))


def test_grid_walk_matches_a_brute_force_caster():
    rng = np.random.default_rng(11)
    compared = hits = excused = 0
    for trial in range(150):
        W, H = int(rng.integers(1, 65)), int(rng.integers(1, 65))
        r = float(rng.uniform(0.05, 1.0))
        x0, y0 = (float(v) for v in rng.uniform(-20.0, 20.0, 2))
        occ = rng.uniform(size=(H, W)) < rng.uniform(0.05, 0.6)
        tab = _table(occ, x0, y0, r)
        faces = _faces(occ, x0, y0, r)
        ext = (x0 - 3 * r, y0 - 3 * r, x0 + (W + 3) * r, y0 + (H + 3) * r)
        n = 64
        sx, sy = rng.uniform(ext[0], ext[2], n), rng.uniform(ext[1], ext[3], n)
        a = rng.uniform(-math.pi, math.pi, n)
        dx, dy = np.cos(a), np.sin(a)
        kind = rng.integers(0, 3, n)
        axis = kind == 1  # axis-parallel beams
        q = rng.integers(0, 4, n)
        dx = np.where(axis, np.array([1.0, -1.0, 0.0, 0.0])[q], dx)
        dy = np.where(axis, np.array([0.0, 0.0, 1.0, -1.0])[q], dy)
        inside = kind == 2  # sensors inside occupied cells
        occ_cells = np.argwhere(occ)
        if len(occ_cells):
            pick = occ_cells[rng.integers(0, len(occ_cells), n)]
            sx = np.where(inside, x0 + (pick[:, 1] + rng.uniform(0.05, 0.95, n)) * r, sx)
            sy = np.where(inside, y0 + (pick[:, 0] + rng.uniform(0.05, 0.95, n)) * r, sy)
        t = map_cast(tab, np.zeros(n, np.int64), sx, sy, dx, dy, np.full(n, 1e9))
        for k in range(n):
            tb, hb, _, _ = cast(sx[k], sy[k], dx[k:k + 1], dy[k:k + 1], np.zeros((0, 4)), faces, 1e9)
            tk = min(t[k], 1e9)
            if _near_corner(x0, y0, r, W, H, sx[k], sy[k], dx[k], dy[k], min(tb[0], tk)):
                excused += 1
                continue
            compared += 1
            assert (hb[0] >= 0) == (t[k] < 1e9), (trial, k)
            if hb[0] >= 0:
                hits += 1
                assert abs(tb[0] - tk) <= 1e-12 * max(1.0, tk), (trial, k, tb[0], tk)
    assert compared > 5000 and hits > 3000 and excused < compared / 10


def test_grid_line_corner_and_outside_conventions():
    """The stated conventions, by hand: a sensor on a grid line lies in the row above it (floor), a beam along that line sees that
    row only; a beam through a corner enters the x-, y- and diagonal neighbours at once; a sensor outside enters through the box; a
    sensor in an occupied cell sees the exit crossing."""
    occ = np.zeros((2, 3), bool)
    occ[0, 1] = True  # cell (1, 0): [1, 2] x [0, 1]
    tab = _table(occ, 0.0, 0.0, 1.0)
    one = lambda sx, sy, dx, dy, lim=1e9: float(map_cast(tab, np.zeros(1, np.int64), np.array([sx]), np.array([sy]), np.array([dx]),
                                                         np.array([dy]), np.array([lim]))[0])
    assert one(-1.0, 0.0, 1.0, 0.0) == 2.0  # along y = 0: row 0, enters cell (1, 0) at x = 1
    assert one(-1.0, 1.0, 1.0, 0.0) == math.inf  # along y = 1: row 1, all free
    assert one(-1.0, 0.5, 1.0, 0.0) == 2.0 and one(5.0, 0.5, -1.0, 0.0) == 3.0  # from outside, both ways
    assert one(-1.0, 0.5, -1.0, 0.0) == math.inf  # looking away from the grid
    assert one(1.5, 0.5, 1.0, 0.0) == 0.5  # inside the occupied cell: the exit
    assert one(1.0, 0.5, -1.0, 0.0) == math.inf  # on its left face (in it, by floor) looking out: the exit at t = 0 does not count
    assert one(-1.0, 0.5, 1.0, 0.0, lim=2.0) == math.inf  # only crossings before lim
    # corners: two diagonal occupied cells; a beam from (0.5, 1.5) along (1, -1) passes the shared corner (1, 1) of (0, 1)...
    diag = np.zeros((2, 2), bool)
    diag[0, 1] = diag[1, 0] = True  # cells (1, 0) and (0, 1)
    tab2 = _table(diag, 0.0, 0.0, 1.0)
    d = math.sqrt(0.5)
    t = map_cast(tab2, np.zeros(1, np.int64), np.array([0.5]), np.array([0.5]), np.array([d]), np.array([d]), np.array([1e9]))[0]
    assert t == 0.5 / d  # from free (0, 0) through the corner (1, 1): the x- and y-neighbours are occupied
    only_diag = np.zeros((2, 2), bool)
    only_diag[1, 1] = True
    t = map_cast(_table(only_diag, 0.0, 0.0, 1.0), np.zeros(1, np.int64), np.array([0.5]), np.array([0.5]), np.array([d]), np.array([d]),
                 np.array([1e9]))[0]
    assert t == 0.5 / d  # the diagonal cell alone counts at the corner


# ---- windowed clearance -------------------------------------------------------------------------------------------------------

def test_windowed_clearance_is_the_brute_force_minimum_up_to_the_window():
    rng = np.random.default_rng(5)
    body0 = np.asarray(Robot(10, 0.1, **DIFF).vertices, np.float64).T
    inside = beyond = 0
    for trial in range(300):
        W, H = int(rng.integers(1, 65)), int(rng.integers(1, 65))
        r = float(rng.uniform(0.05, 1.0))
        x0, y0 = (float(v) for v in rng.uniform(-10.0, 10.0, 2))
        occ = rng.uniform(size=(H, W)) < rng.uniform(0.01, 0.3)
        if not occ.any():
            continue
        tab = _table(occ, x0, y0, r)
        s = (float(rng.uniform(x0 - 3, x0 + W * r + 3)), float(rng.uniform(y0 - 3, y0 + H * r + 3)), float(rng.uniform(-math.pi, math.pi)))
        body = ow.robot_polygon(s, body0)
        window = float(rng.uniform(0.05, 3.0))
        jj, ii = np.nonzero(occ)
        Q = cell_polygons(tab, 0, ii, jj)
        brute = float(clearance_robot_pairs(np.ascontiguousarray(np.broadcast_to(np.asarray(body)[None], (len(Q), 4, 2))), Q).min())
        got = map_clearance(tab, 0, body, window)
        if brute <= window:
            inside += 1
            assert got == brute, (trial, got, brute)
        else:
            beyond += 1
            assert got == window, (trial, got, window)
    assert inside > 50 and beyond > 50


# ---- builders -----------------------------------------------------------------------------------------------------------------

def _free_cells_reachable(occ, a, b):
    """4-connected free path between cells a and b (j, i)?"""
    from neupan_b200.world import _bfs
    dist, _ = _bfs(~occ, a)
    return dist[b] >= 0


def _cell_of(m, p):
    return int(math.floor((p[1] - m["origin"][1]) / m["resolution"])), int(math.floor((p[0] - m["origin"][0]) / m["resolution"]))


@pytest.mark.parametrize("builder", ["maze", "cave"])
def test_builders_are_deterministic_and_start_free(lib, builder):
    make = maze if builder == "maze" else cave
    a, b = make(6, seed=3), make(6, seed=3)
    for x, y in zip(a, b):
        assert np.array_equal(x["map"]["occupancy"], y["map"]["occupancy"]) and x["start"] == y["start"] and x["goal"] == y["goal"]
        assert np.array_equal(x["path"], y["path"])
    assert not np.array_equal(a[0]["map"]["occupancy"], a[1]["map"]["occupancy"])  # one layout per environment by default
    assert np.array_equal(make(6, seed=3)[4:][0]["map"]["occupancy"], a[4]["map"]["occupancy"])  # seeded per layout
    shared = make(6, seed=3, layouts=2)
    assert shared[0]["map"]["occupancy"] is shared[2]["map"]["occupancy"] and len(pack_maps(shared)[0]) == 2
    cfg = make_config(Robot(10, 0.1, **DIFF), LIDAR, 0.1, max_envs=64)
    assert _check(lib, cfg, make(16, seed=7)) == _lib.NB_OK  # every start body is free
    for sc in a:  # the path's points lie in free cells, and start and goal are joined through free cells
        m = sc["map"]
        occ = m["occupancy"]
        cells = [_cell_of(m, p) for p in sc["path"][:, :2]]
        assert not any(occ[c] for c in cells)
        assert _free_cells_reachable(occ, _cell_of(m, sc["start"]), _cell_of(m, sc["goal"]))
        assert np.allclose(sc["path"][0, :3], sc["start"]) and np.allclose(sc["path"][-1, :2], sc["goal"])


def test_maze_is_solvable_at_every_seed_and_closed():
    for seed in range(20):
        for sc in maze(2, cells=(int(3 + seed % 4), int(4 + seed % 3)), seed=seed):
            m = sc["map"]
            occ = m["occupancy"]
            assert _free_cells_reachable(occ, _cell_of(m, sc["start"]), _cell_of(m, sc["goal"])), seed
            from neupan_b200.world import _bfs
            dist, _ = _bfs(~occ, _cell_of(m, sc["start"]))
            assert (dist[0] < 0).all() and (dist[-1] < 0).all() and (dist[:, 0] < 0).all() and (dist[:, -1] < 0).all()  # closed border
            assert not any(occ[_cell_of(m, p)] for p in sc["path"][:, :2])
