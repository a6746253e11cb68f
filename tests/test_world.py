"""The batched world's CPU side: the oracle's ray casts, clearances and motion on hand-built cases with known answers, its scans
through the scan -> points oracle, and the host validation of scenes and configs (no device needed)."""
import ctypes as C
import math

import numpy as np
import pytest

from neupan_b200 import _lib, build as nb_build
from neupan_b200.robot import robot as Robot
from neupan_b200.synth import rollout as synth_rollout
from neupan_b200.world import corridor, dyna_obs, make_config, pack_scenes, rectangle
from oracle import scan as oscan, world as ow

LIDAR = dict(angle_min=-math.pi, angle_max=math.pi, range_min=0.0, range_max=10.0, number=360)


@pytest.fixture(scope="module")
def lib():
    nb_build.build()
    return _lib.load()


def _cfg(kin="diff", lidar=LIDAR, dt=0.1, L=None, vertices=None):
    rb = Robot(10, dt, kinematics=kin, length=1.6, width=2.0, wheelbase=L, vertices=vertices)
    return dict(kinematics=kin, step_time=dt, wheelbase=L, angle_min=lidar["angle_min"], angle_max=lidar["angle_max"],
                range_max=lidar["range_max"], number=lidar["number"], scan_offset=lidar.get("scan_offset", (0.0, 0.0, 0.0)),
                robot_vertices=np.asarray(rb.vertices, np.float64).T), rb


def _scene(obstacles, start=(0.0, 0.0, 0.0), bounds=(-50.0, -50.0, 50.0, 50.0), goal=(100.0, 100.0), thr=0.1):
    return dict(obstacles=obstacles, bounds=bounds, start=start, goal=goal, goal_threshold=thr)


def _cast_one(obstacles, direction=0.0, origin=(0.0, 0.0), range_max=10.0):
    """One beam from origin along the world angle `direction` through the oracle's env scan."""
    cfg, _ = _cfg(lidar=dict(angle_min=direction, angle_max=direction, range_min=0.0, range_max=range_max, number=1))
    w = ow.OracleWorld(cfg, pack_scenes([_scene(obstacles, start=(origin[0], origin[1], 0.0))]))
    r, v, hit, tie, tan_ = w.scan()
    return r[0, 0], hit[0, 0], v[0, :, 0], tan_[0, 0]


def test_head_on_circle_is_at_distance_minus_radius():
    r, hit, v, _ = _cast_one([dict(center=(5.0, 0.0), radius=1.5, velocity=(0.25, -0.5))])
    assert r == 3.5 and hit == 0 and tuple(v) == (0.25, -0.5)


def test_grazing_ray_touches_and_a_slightly_smaller_circle_is_missed():
    r, hit, _, tangent = _cast_one([dict(center=(5.0, 1.0), radius=1.0)])
    assert r == 5.0 and hit == 0 and tangent  # discriminant exactly 0: the tangent point counts as a crossing
    r, hit, v, _ = _cast_one([dict(center=(5.0, 1.0), radius=0.999)])
    assert r == 10.0 and hit == -1 and tuple(v) == (0.0, 0.0)


def test_ray_through_a_polygon_vertex():
    diamond = [[-1.0, 0.0], [0.0, -1.0], [1.0, 0.0], [0.0, 1.0]]
    r, hit, _, _ = _cast_one([dict(center=(6.0, 0.0), vertices=diamond)])
    assert r == 5.0 and hit == 0
    # the lower index wins an exact tie: a circle touching the same vertex, listed second
    r, hit, _, _ = _cast_one([dict(center=(6.0, 0.0), vertices=diamond), dict(center=(4.0, 0.0), radius=1.0)])
    assert r == 3.0 and hit == 1
    r, hit, _, _ = _cast_one([dict(center=(4.0, 0.0), radius=1.0), dict(center=(6.0, 0.0), vertices=diamond)])
    assert r == 3.0 and hit == 0


def test_sensor_inside_an_obstacle_sees_the_exit_crossing():
    r, hit, _, _ = _cast_one([dict(center=(0.5, 0.0), radius=2.0)])
    assert r == 2.5 and hit == 0
    r, hit, _, _ = _cast_one([dict(center=(1.0, 0.0), vertices=rectangle(6.0, 2.0))])
    assert r == 4.0 and hit == 0


def test_miss_and_beyond_range_return_range_max():
    assert _cast_one([])[:2] == (10.0, -1)
    assert _cast_one([dict(center=(0.0, 5.0), radius=1.0)])[:2] == (10.0, -1)      # off the beam
    assert _cast_one([dict(center=(-5.0, 0.0), radius=1.0)])[:2] == (10.0, -1)     # behind the sensor
    assert _cast_one([dict(center=(11.0, 0.0), radius=1.0)])[:2] == (10.0, -1)     # t = 10 = range_max is a miss


def test_beam_angles_are_the_linspace_of_the_lidar():
    for R, lo, hi in ((1, -0.3, 0.3), (37, -math.pi, math.pi), (100, -math.pi / 2, math.pi / 2)):
        ca, sa = ow.beam_table(lo, hi, R)
        a = np.linspace(lo, hi, R)
        assert np.array_equal(ca, np.cos(a)) or np.abs(ca - np.cos(a)).max() < 1e-15
        assert np.abs(np.arctan2(sa, ca) - a).max() < 1e-15
    # a robot turned by theta with a sensor turned by off_th: beam i points at theta + off_th + a_i
    cfg, _ = _cfg(lidar=dict(LIDAR, number=8, scan_offset=(0.0, 0.0, 0.4)))
    w = ow.OracleWorld(cfg, pack_scenes([_scene([dict(center=(0.0, 0.0), radius=3.0)], start=(0.0, 0.0, 0.3))]))
    r, _, hit, _, _ = w.scan()
    assert np.allclose(r, 3.0, atol=1e-15) and (hit == 0).all()


def _boundary_distance(p, scene):
    d = math.inf
    for ob in scene["obstacles"]:
        cx, cy = ob["center"]
        if "vertices" in ob:
            v = np.asarray(ob["vertices"]) + (cx, cy)
            for k in range(len(v)):
                a, b = v[k], v[(k + 1) % len(v)]
                d = min(d, ow.seg_dist(p[0], p[1], a[0], a[1], b[0], b[1]))
        else:
            d = min(d, abs(math.hypot(p[0] - cx, p[1] - cy) - ob["radius"]))
    return d


@pytest.mark.parametrize("offset", [(0.0, 0.0, 0.0), (0.3, -0.1, 0.2)])
def test_oracle_scans_map_to_points_on_the_obstacle_boundaries(offset):
    scenes = corridor(3, seed=5) + dyna_obs(3, seed=6)
    rng = np.random.default_rng(0)
    for sc in scenes:  # robots somewhere inside the scene, turned at random
        sc["start"] = (sc["start"][0] + rng.uniform(5, 25), sc["start"][1] + rng.uniform(-0.5, 0.5), rng.uniform(-np.pi, np.pi))
    lidar = dict(LIDAR, number=181, scan_offset=offset)
    cfg, _ = _cfg(lidar=lidar)
    w = ow.OracleWorld(cfg, pack_scenes(scenes))
    ranges = w.scan()[0]
    n = 0
    for b, sc in enumerate(scenes):
        pts = oscan.scan_to_point(w.states[b].reshape(3, 1), dict(lidar, ranges=ranges[b]), scan_offset=offset)
        for p in pts.T:
            assert _boundary_distance(p, sc) < 1e-9
            n += 1
    assert n > 200


def test_clearance_hand_built_cases():
    sq = [(0.0, 0.0), (2.0, 0.0), (2.0, 2.0), (0.0, 2.0)]  # robot: the square [0, 2]^2
    assert ow.clearance_circle(sq, 5.0, 1.0, 1.0) == 2.0          # separated
    assert ow.clearance_circle(sq, 3.0, 1.0, 1.0) == 0.0          # touching
    assert ow.clearance_circle(sq, 2.5, 1.0, 1.0) == 0.0          # overlapping
    assert ow.clearance_circle(sq, 1.0, 1.0, 0.1) == 0.0          # centre inside the robot
    assert ow.clearance_circle(sq, 1.0, 1.0, 9.0) == 0.0          # circle around the robot
    assert abs(ow.clearance_circle(sq, 5.0, 6.0, 1.0) - 4.0) < 1e-15  # nearest feature: the corner (2, 2), distance 5
    # polygons: separated along x, diagonal (vertex-vertex), touching, overlapping, one inside the other
    shift = lambda P, dx, dy: [(x + dx, y + dy) for x, y in P]
    assert ow.clearance_polygon(sq, shift(sq, 3.0, 0.5)) == 1.0
    assert abs(ow.clearance_polygon(sq, shift(sq, 5.0, 6.0)) - 5.0) < 1e-15
    assert ow.clearance_polygon(sq, shift(sq, 2.0, 0.0)) == 0.0
    assert ow.clearance_polygon(sq, shift(sq, 1.0, 1.0)) == 0.0
    assert ow.clearance_polygon(sq, [(0.5, 0.5), (1.5, 0.5), (1.0, 1.5)]) == 0.0
    # only an edge normal of the triangle separates them (SAT on the obstacle's axes): distance = from (2, 2) to the hypotenuse
    tri = [(3.0, 2.0), (2.0, 3.0), (4.0, 4.0)]
    assert not ow._separated(sq, tri) and ow._separated(tri, sq)
    assert abs(ow.clearance_polygon(sq, tri) - math.sqrt(0.5)) < 1e-15


@pytest.mark.parametrize("kin", ["diff", "acker", "omni"])
def test_one_step_of_each_motion_model_equals_synth_rollout(kin):
    rng = np.random.default_rng(11)
    L = 3.0 if kin == "acker" else None
    s0 = np.column_stack([rng.uniform(-5, 5, (64, 2)), rng.uniform(-np.pi, np.pi, 64)])
    u = np.column_stack([rng.uniform(-2, 4, 64), rng.uniform(-0.6, 0.6, 64)]).astype(np.float32).astype(np.float64)
    ref = synth_rollout(kin, s0, u[:, :, None], 0.1, L)[:, :, 1]
    act = u if kin != "omni" else np.column_stack([u[:, 0] * np.cos(u[:, 1]), u[:, 0] * np.sin(u[:, 1])])  # PlannerBatch's (vx, vy)
    got = np.array([ow.integrate(kin, s0[b], act[b], 0.1, L) for b in range(64)])
    assert np.abs(got - ref).max() <= 1e-14


def test_reflection_keeps_moving_centres_inside_their_rectangle():
    scenes = dyna_obs(8, seed=3)
    cfg, _ = _cfg()
    w = ow.OracleWorld(cfg, pack_scenes(scenes))
    w.obs[:, 2:4] *= 4.0  # 2 m/s: many bounces in 200 steps
    speed0 = np.hypot(w.obs[:, 2], w.obs[:, 3])
    flips = 0
    for _ in range(200):
        v_before = w.obs[:, 2:4].copy()
        w.step(np.zeros((8, 2)))
        flips += int((np.sign(v_before) != np.sign(w.obs[:, 2:4])).sum())
        for b in range(8):
            o = slice(w.obs_begin[b], w.obs_begin[b + 1])
            lo, hi = w.env[b, 0:2], w.env[b, 2:4]
            assert (w.obs[o, 0:2] >= lo).all() and (w.obs[o, 0:2] <= hi).all()
    assert flips > 50 and np.array_equal(np.hypot(w.obs[:, 2], w.obs[:, 3]), speed0)


def test_collision_is_sticky_and_freezes_the_robot():
    cfg, _ = _cfg()
    w = ow.OracleWorld(cfg, pack_scenes([_scene([dict(center=(2.5, 0.0), radius=0.5)], start=(0.0, 0.0, 0.0), goal=(3.0, 0.0), thr=0.5)]))
    col, arr, clear = w.step(np.array([[5.0, 0.0]]))  # the robot's front moves from x = 0.8 to 1.3: clearance 0.7
    assert col[0] == 0 and abs(clear[0] - 0.7) < 1e-12
    col, arr, clear = w.step(np.array([[8.0, 0.0]]))  # front at 2.1 > 2.0: overlap
    assert col[0] == 1 and clear[0] == 0.0
    x = w.states[0].copy()
    w.step(np.array([[8.0, 0.0]]))
    assert np.array_equal(w.states[0], x) and w.collided[0] == 1 and w.arrived[0] == 0


def test_world_config_struct_layout_matches_header():
    # nb_world_config: 6 int32, then 5 + 3 + 16 doubles
    assert C.sizeof(_lib.WorldConfig) == 6 * 4 + 24 * 8
    assert _lib.WorldConfig.step_time.offset == 24 and _lib.WorldConfig.range_max.offset == 56
    assert _lib.WorldConfig.scan_offset.offset == 64 and _lib.WorldConfig.robot_vertices.offset == 88


def _check(lib, cfg, packed, B=None):
    B = len(packed[0]) - 1 if B is None else B
    return lib.nb_world_check_scenes(C.byref(cfg), B, *[C.c_void_p(a.ctypes.data) for a in packed])


def test_host_validation_rejects_bad_scenes_without_a_device(lib):
    rb = Robot(10, 0.1, kinematics="diff", length=1.6, width=2.0)
    cfg = make_config(rb, LIDAR, 0.1, max_envs=4)
    ok = pack_scenes(dyna_obs(2, seed=1))
    assert _check(lib, cfg, ok) == _lib.NB_OK
    assert _check(lib, cfg, ok, B=5) == _lib.NB_ERR_INVALID  # above max_envs

    def bad(scene, what):
        assert _check(lib, cfg, pack_scenes([scene])) == _lib.NB_ERR_INVALID, what
        return lib.nb_last_error().decode()

    circ = lambda n: [dict(center=(0.0, 0.0), radius=1.0)] * n
    octagon = [[math.cos(k * math.pi / 4), math.sin(k * math.pi / 4)] for k in range(8)]
    assert _check(lib, cfg, pack_scenes([_scene(circ(256))])) == _lib.NB_OK
    assert "257 obstacles" in bad(_scene(circ(257)), "too many obstacles")
    assert _check(lib, cfg, pack_scenes([_scene([dict(center=(0.0, 0.0), vertices=octagon)] * 256)])) == _lib.NB_OK  # 2048 edges
    # (256 obstacles of at most 8 vertices: the 2048-edge limit of an environment cannot be exceeded)
    assert "9 vertices" in bad(_scene([dict(center=(0.0, 0.0), vertices=[[math.cos(k * 0.7), math.sin(k * 0.7)] for k in range(9)])]), "nonagon")
    assert "convex" in bad(_scene([dict(center=(0.0, 0.0), vertices=[[0, 0], [2, 0], [1, 0.2], [1, 2]])]), "reflex vertex")
    assert "convex" in bad(_scene([dict(center=(0.0, 0.0), vertices=[[0, 0], [1, 0], [2, 0]])]), "degenerate")
    assert "radius" in bad(_scene([dict(center=(0.0, 0.0), radius=0.0)]), "zero radius")
    assert "outside" in bad(_scene([dict(center=(60.0, 0.0), radius=1.0, velocity=(0.1, 0.0))]), "moving centre outside")
    assert "exceeds" in bad(_scene([dict(center=(0.0, 0.0), radius=1.0, velocity=(2000.0, 0.0))]), "too fast")
    assert "rectangle" in bad(_scene([], bounds=(1.0, 0.0, 0.0, 1.0)), "empty rectangle")
    # ragged offsets that do not add up
    ob, rows, vb, verts, envs = pack_scenes(dyna_obs(2, seed=1))
    for broken in (np.array([1, 20, 40], np.int32), np.array([0, 30, 20], np.int32)):
        assert _check(lib, cfg, (broken, rows, vb, verts, envs)) == _lib.NB_ERR_INVALID
    vb_bad = vb.copy(); vb_bad[3] = 2  # obstacle 2 gets 2 vertices
    assert _check(lib, cfg, (ob, rows, vb_bad, np.zeros((4, 2)), envs)) == _lib.NB_ERR_INVALID
    assert "vertices" in lib.nb_last_error().decode()


def test_world_create_rejects_bad_configs_before_touching_the_device(lib):
    rb = Robot(10, 0.1, kinematics="diff", length=1.6, width=2.0)
    h = C.c_void_p()
    for field, value, text in (("num_beams", 0, "R >= 1"), ("step_time", 0.0, "step_time"), ("range_max", -1.0, "range_max"),
                               ("robot_num_vertices", 2, "robot polygon"), ("kinematics", 3, "kinematics")):
        cfg = make_config(rb, LIDAR, 0.1, max_envs=4)
        setattr(cfg, field, value)
        assert lib.nb_world_create(C.byref(cfg), C.byref(h)) == _lib.NB_ERR_INVALID
        assert text in lib.nb_last_error().decode()
    cfg = make_config(Robot(10, 0.1, kinematics="acker", length=4.6, width=1.6, wheelbase=3), LIDAR, 0.1, max_envs=4)
    cfg.wheelbase = 0.0
    assert lib.nb_world_create(C.byref(cfg), C.byref(h)) == _lib.NB_ERR_INVALID
    cfg = make_config(rb, LIDAR, 0.1, max_envs=4)
    cfg.robot_vertices[2], cfg.robot_vertices[3] = 0.0, 0.0  # a reflex robot polygon
    assert lib.nb_world_create(C.byref(cfg), C.byref(h)) == _lib.NB_ERR_INVALID
    for fn, args in ((lib.nb_world_scan, (None, 1, None, None, None, None)), (lib.nb_world_step, (None, 1, None, None, None, None, None)),
                     (lib.nb_world_read_state, (None, 1, None, None, None, None, None)), (lib.nb_world_set_scenes, (None, 1, None, None, None, None, None))):
        assert fn(*args) == _lib.NB_ERR_INVALID


def test_scene_builders_are_seeded_per_environment():
    a, b = dyna_obs(6, seed=9), dyna_obs(3, seed=9)
    for x, y in zip(a[:3], b):
        assert x["start"] == y["start"] and all(np.array_equal(np.asarray(p["center"]), np.asarray(q["center"])) for p, q in zip(x["obstacles"], y["obstacles"]))
    sc = dyna_obs(50, seed=2)
    speeds = [math.hypot(*o["velocity"]) for s in sc for o in s["obstacles"]]
    radii = [o["radius"] for s in sc for o in s["obstacles"]]
    assert max(speeds) <= 0.5 and 0.4 <= min(radii) and max(radii) <= 1.0 and all(len(s["obstacles"]) == 20 for s in sc)
    c = corridor(2, seed=0, circles=0)
    assert len(c[0]["obstacles"]) == 2 and c[0]["path"][-1, 0] == 60.0
