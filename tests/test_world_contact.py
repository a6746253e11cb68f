"""Obstacle contact on the CPU (no device needed): the refusals of nb_world_check_obstacle_contact, the scene builders with and
without ``contact``, the contact predicate of tests/world_contact_oracle.py against an independent brute-force formulation (and its
symmetry), and an invariant run in which no moving obstacle ever touches another one."""
import ctypes as C
import hashlib
import math

import numpy as np
import pytest

from neupan_b200 import _lib, build as nb_build
from neupan_b200.robot import robot as Robot
from neupan_b200.world import (cave, dyna_non_obs, dyna_obs, make_config, maze, pack_behaviors, pack_map_contact, pack_maps,
                               pack_obstacle_contact, pack_scenes_ex, random_outline)
from world_contact_oracle import ContactOracleWorld, footprints_touch, touches

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


def _behaviors(scenes):
    return pack_behaviors(scenes) if any("behavior" in ob for sc in scenes for ob in sc["obstacles"]) else None


def _oracle(scenes, seed=0):
    maps = pack_maps(scenes) if any("map" in sc for sc in scenes) else None
    block = pack_map_contact(scenes) if maps is not None else None
    return ContactOracleWorld(_cfg(), pack_scenes_ex(scenes), _behaviors(scenes), seed, maps=maps, block=block,
                              contact=pack_obstacle_contact(scenes))


def _check(lib, scenes, flags=None):
    cfg = make_config(_robot(), LIDAR, DT, max_envs=max(8, len(scenes)))
    packed = pack_scenes_ex(scenes)
    beh = _behaviors(scenes)
    flags = pack_obstacle_contact(scenes) if flags is None else np.asarray(flags, np.int32)
    return lib.nb_world_check_obstacle_contact(C.byref(cfg), len(scenes), *[C.c_void_p(a.ctypes.data) for a in packed],
                                               C.c_void_p(beh.ctypes.data) if beh is not None else None,
                                               C.c_void_p(flags.ctypes.data) if flags is not None else None)


def _scene(obstacles, contact=True):
    sc = dict(obstacles=obstacles, bounds=(0.0, 0.0, 20.0, 20.0), start=(1.0, 1.0, 0.0), goal=(19.0, 19.0), goal_threshold=0.3, path=None)
    if contact:
        sc["obstacle_contact"] = True
    return sc


SQUARE = [[-1.0, -1.0], [1.0, -1.0], [1.0, 1.0], [-1.0, 1.0]]
NOTCH = [[-2.0, -2.0], [2.0, -2.0], [2.0, 2.0], [0.5, 2.0], [0.5, -0.5], [-0.5, -0.5], [-0.5, 2.0], [-2.0, 2.0]]  # a U, open upwards


# ---- refusals ---------------------------------------------------------------------------------------------------------------

def test_refusals_name_the_environment_and_obstacle(lib):
    ok = [_scene([dict(center=(5.0, 5.0), radius=1.0, velocity=(0.5, 0.0)), dict(center=(7.5, 5.0), radius=1.0),
                  dict(center=(15.0, 15.0), vertices=SQUARE), dict(center=(15.5, 15.0), radius=1.0)]),  # two static ones overlap
          _scene([dict(center=(5.0, 5.0), radius=1.0, velocity=(0.5, 0.0)), dict(center=(6.0, 5.0), radius=1.0)], contact=False)]
    assert _check(lib, ok) == _lib.NB_OK, lib.nb_last_error()

    def refused(rc, msg):
        assert rc == _lib.NB_ERR_INVALID
        assert msg in lib.nb_last_error().decode(), lib.nb_last_error().decode()

    refused(_check(lib, ok, flags=[2, 0]), "environment 0: obstacle contact flag 2 (0 or 1)")
    refused(_check(lib, ok, flags=[0, -1]), "environment 1: obstacle contact flag -1 (0 or 1)")
    refused(_check(lib, ok, flags=[1, 1]), "environment 1, obstacle 4: moves but its start footprint overlaps or touches obstacle 5")
    cfg = make_config(_robot(), LIDAR, DT, max_envs=8)
    packed = pack_scenes_ex(ok)
    refused(lib.nb_world_check_obstacle_contact(C.byref(cfg), 2, *[C.c_void_p(a.ctypes.data) for a in packed], None, None), "null flags")
    # exactly touching counts; each pair of kinds; a reactive obstacle at rest counts as a mover
    touching = [
        [dict(center=(5.0, 5.0), radius=1.0, velocity=(0.1, 0.0)), dict(center=(7.0, 5.0), radius=1.0)],
        [dict(center=(5.0, 5.0), radius=1.0), dict(center=(7.0, 5.0), vertices=SQUARE, velocity=(0.0, 0.1))],
        [dict(center=(5.0, 5.0), vertices=SQUARE, velocity=(0.1, 0.0)), dict(center=(7.0, 6.5), vertices=SQUARE)],
        [dict(center=(5.0, 5.0), outline=NOTCH, velocity=(0.1, 0.0)), dict(center=(5.0, 4.0), radius=0.2)],  # inside the U's floor
        [dict(center=(5.0, 5.0), outline=NOTCH), dict(center=(8.0, 5.0), vertices=SQUARE, velocity=(0.1, 0.0))],  # edge on edge at x = 7
        [dict(center=(5.0, 5.0), outline=NOTCH), dict(center=(5.0, 9.0), outline=NOTCH, velocity=(0.1, 0.0))],  # edges share y = 7
        [dict(center=(5.0, 5.0), radius=1.0, velocity=(0.0, 0.0), behavior=dict(name="rvo", vxmax=0.5, vymax=0.5)),
         dict(center=(6.0, 5.0), radius=1.0)],
    ]
    for i, obs in enumerate(touching):
        rc = _check(lib, [_scene(obs)])
        refused(rc, "environment 0, obstacle")
    # the circle in the U's notch, clear of its walls, is accepted
    assert _check(lib, [_scene([dict(center=(5.0, 5.0), outline=NOTCH), dict(center=(5.0, 6.0), radius=0.4, velocity=(0.0, 0.1))])]) == _lib.NB_OK


# ---- builders ---------------------------------------------------------------------------------------------------------------

def _fingerprint(scenes):
    h = hashlib.sha256()
    for sc in scenes:
        h.update(np.ascontiguousarray(sc["path"]).tobytes())
        for ob in sc["obstacles"]:
            h.update(repr(sorted((k, v if k not in ("outline", "vertices") else np.asarray(v, np.float64).tobytes()) for k, v in ob.items())).encode())
        h.update(repr(sorted((k, v) for k, v in sc.items() if k not in ("obstacles", "path", "map"))).encode())
        if "map" in sc:
            h.update(np.ascontiguousarray(sc["map"]["occupancy"]).tobytes())
            h.update(repr(sorted((k, v) for k, v in sc["map"].items() if k != "occupancy")).encode())
    return h.hexdigest()


def test_builders_without_contact_are_unchanged():
    # the scenes these builders made before they took contact
    assert _fingerprint(dyna_obs(3, seed=4, contact=False)) == "5aac81eed924a2afca8de111b428e1ac7e41f7482f98ab1e3d2b98a645a7beda"
    assert _fingerprint(dyna_obs(3, seed=4, behavior="rvo")) == "3947df22fd162aaedee2f732a6a7cd8bb539e2dee1a33f24aabd1abf4b63486a"
    assert _fingerprint(dyna_non_obs(3, seed=5, contact=False)) == "67346fe30bcd2110f40ea528826adf21b838dc2c365ed9d4acac9074f7a48682"
    assert _fingerprint(dyna_non_obs(3, seed=5, behavior="rvo")) == "c9bf393b0e6e6ae9bfff60d3eaa267096f3df14417e89a36dff05fdae8caffe3"
    assert _fingerprint(maze(2, seed=1, movers=8, contact=False)) == "b416330360d27e6e32ccba4cbdda68242f31ba031294e238e95ba6ee191eeccb"
    assert (_fingerprint(cave(2, seed=2, size=(20.0, 20.0), movers=12, behavior="rvo", contact=False))
            == "0996f234973a4611e8f27bf80fb3fa2217106acd6031ffa9e76b1b64a0e82d4b")


def test_builders_with_contact_are_deterministic_and_start_apart(lib):
    builds = [lambda: dyna_obs(16, seed=3, contact=True), lambda: dyna_obs(16, seed=3, behavior="rvo", contact=True),
              lambda: dyna_non_obs(16, seed=3, contact=True), lambda: dyna_non_obs(16, seed=3, behavior="rvo", contact=True),
              lambda: maze(4, seed=1, movers=8, contact=True), lambda: cave(3, seed=2, movers=12, behavior="rvo", contact=True)]
    for make in builds:
        scenes = make()
        assert _fingerprint(scenes) == _fingerprint(make())
        assert all(sc["obstacle_contact"] for sc in scenes)
        assert _check(lib, scenes) == _lib.NB_OK, lib.nb_last_error()
        o = _oracle(scenes)
        assert o.touching_pairs() == []
    plain = dyna_obs(16, seed=3)
    contact = dyna_obs(16, seed=3, contact=True)
    # only the centres of overlapping circles change, and some do
    changed = sum(a["center"] != b["center"] for sa, sb in zip(plain, contact) for a, b in zip(sa["obstacles"], sb["obstacles"]))
    assert changed > 0
    for sa, sb in zip(plain, contact):
        for a, b in zip(sa["obstacles"], sb["obstacles"]):
            assert a["radius"] == b["radius"] and a["velocity"] == b["velocity"]


# ---- the predicate ----------------------------------------------------------------------------------------------------------

def _point_seg(x, a, b):
    """Distances from the points x (..., 2) to the segments a-b (..., 2) by projection, broadcast."""
    e, w = b - a, x - a
    t = np.clip((w * e).sum(-1) / (e * e).sum(-1), 0.0, 1.0)
    return np.linalg.norm(w - t[..., None] * e, axis=-1)


def _brute_seg_seg(P, Q):
    """The smallest distance between an edge of the closed polygon P (m, 2) and one of Q (n, 2): 0 where two edges' parametric
    solution lies in both, else the smallest endpoint-to-segment distance, over all m n edge pairs."""
    p, q = P[:, None, :], np.roll(P, -1, 0)[:, None, :]
    a, b = Q[None, :, :], np.roll(Q, -1, 0)[None, :, :]
    u, v, w = q - p, b - a, a - p
    den = u[..., 0] * v[..., 1] - u[..., 1] * v[..., 0]
    with np.errstate(divide="ignore", invalid="ignore"):
        s = (w[..., 0] * v[..., 1] - w[..., 1] * v[..., 0]) / den
        t = (w[..., 0] * u[..., 1] - w[..., 1] * u[..., 0]) / den
    if ((den != 0.0) & (s >= 0.0) & (s <= 1.0) & (t >= 0.0) & (t <= 1.0)).any():
        return 0.0
    p, q, a, b = np.broadcast_arrays(p, q, a, b)
    return float(min(_point_seg(p, a, b).min(), _point_seg(q, a, b).min(), _point_seg(a, p, q).min(), _point_seg(b, p, q).min()))


def _winding(poly, x):
    """Winding number of the closed polygon about x (sum of the turned angles)."""
    d = poly - x
    ang = np.arctan2(d[:, 1], d[:, 0])
    turn = np.diff(np.concatenate([ang, ang[:1]]))
    turn = (turn + np.pi) % (2.0 * np.pi) - np.pi
    return int(round(turn.sum() / (2.0 * np.pi)))


def _brute_gap(sa, ca, sb, cb):
    """Signed gap of two footprints: the boundary distance (minus the radii of circles), negative when one contains a point of
    the other."""
    def pts(s, c):
        return None if s[0] == "circle" else np.asarray(s[1], np.float64) + np.asarray(c, np.float64)
    pa, pb = pts(sa, ca), pts(sb, cb)
    ca, cb = np.asarray(ca, np.float64), np.asarray(cb, np.float64)
    if pa is None and pb is None:
        return float(np.linalg.norm(ca - cb)) - sa[1] - sb[1]
    if pa is None or pb is None:
        (c, r), poly = ((ca, sa[1]), pb) if pa is None else ((cb, sb[1]), pa)
        d = float(_point_seg(c[None], poly, np.roll(poly, -1, 0)).min())
        return -1.0 if _winding(poly, c) != 0 else d - r
    if _winding(pb, pa[0]) != 0 or _winding(pa, pb[0]) != 0:
        return -1.0
    return _brute_seg_seg(pa, pb)


def _random_shape(rng, kind):
    if kind == "circle":
        return "circle", float(rng.uniform(0.2, 1.5))
    if kind == "convex":
        n = int(rng.integers(3, 9))
        a = np.sort(rng.uniform(0.0, 2.0 * np.pi, n))
        while np.diff(np.concatenate([a, a[:1] + 2.0 * np.pi])).max() >= np.pi:
            a = np.sort(rng.uniform(0.0, 2.0 * np.pi, n))
        return "convex", np.stack([np.cos(a), np.sin(a)], 1) * rng.uniform(0.3, 1.5)  # on a circle: convex
    return "outline", random_outline(rng, rng.uniform(0.5, 1.5), 0.9, rng.uniform(0.0, 1.0), int(rng.integers(4, 17)))


KIND_PAIRS = [("circle", "circle"), ("circle", "convex"), ("circle", "outline"), ("convex", "convex"), ("convex", "outline"),
              ("outline", "outline")]


def test_predicate_matches_brute_force_and_is_symmetric():
    """1800 pairs of each of the six kind pairs (10800 in all): a third placed at random, two thirds moved along a random direction
    to within 1e-3 .. 1e-11 m of touching (bisection on the brute-force gap), on either side.  The oracle's predicate (broad phase
    included) equals the brute force except within 1e-12 of touching, and touches(i, j) == touches(j, i) everywhere."""
    rng = np.random.default_rng(11)
    excused, total, near, hits = 0, 0, 0, 0
    for ka, kb in KIND_PAIRS:
        for q in range(1800):
            sa, sb = _random_shape(rng, ka), _random_shape(rng, kb)
            ca = tuple(rng.uniform(-10.0, 10.0, 2))
            u = rng.normal(size=2)
            u /= np.linalg.norm(u)
            if q % 3 == 0:
                cb = tuple(np.asarray(ca) + u * rng.uniform(0.0, 4.0))
            else:  # the touching distance along u: far is clear, at the centre they overlap
                lo, hi = 0.0, 8.0
                for _ in range(60):
                    mid = 0.5 * (lo + hi)
                    if _brute_gap(sa, ca, sb, tuple(np.asarray(ca) + u * mid)) > 0.0:
                        hi = mid
                    else:
                        lo = mid
                off = float(10.0 ** rng.uniform(-11.0, -3.0)) * (1.0 if q % 3 == 1 else -1.0)
                cb = tuple(np.asarray(ca) + u * (hi + off))
                near += 1
            gap = _brute_gap(sa, ca, sb, cb)
            t = touches(sa, ca, sb, cb)
            assert t == touches(sb, cb, sa, ca) == footprints_touch(sb, cb, sa, ca), (ka, kb, q)
            total += 1
            hits += t
            if gap != 0.0 and abs(gap) <= 1e-12:  # 0: two edges cross
                excused += 1
                continue
            assert t == (gap <= 0.0), (ka, kb, q, gap, sa, ca, sb, cb)
    assert total >= 10_000 and near >= 7000 and 0.3 * total < hits < 0.7 * total
    assert excused < total // 100


# ---- the invariant ----------------------------------------------------------------------------------------------------------

def _crowded(rng, n, box, reactive_every=0):
    """n obstacles of all three kinds, placed apart (circumcircles) in box, speeds up to 0.5 m/s, every reactive_every-th one reactive."""
    obs = []
    x0, y0, x1, y1 = box
    while len(obs) < n:
        kind = ("circle", "convex", "outline")[len(obs) % 3]
        c = (float(rng.uniform(x0 + 1, x1 - 1)), float(rng.uniform(y0 + 1, y1 - 1)))
        if kind == "circle":
            ob, r = dict(center=c, radius=float(rng.uniform(0.2, 0.6))), None
        elif kind == "convex":
            ob = dict(center=c, vertices=(np.asarray(SQUARE) * rng.uniform(0.2, 0.5)).tolist())
        else:
            ob = dict(center=c, outline=random_outline(rng, rng.uniform(0.3, 0.6), 0.9, 0.5, int(rng.integers(4, 10))))
        rad = ob.get("radius") or float(np.hypot(*np.asarray(ob.get("vertices", ob.get("outline")), np.float64).T).max())
        if any(math.hypot(c[0] - p["center"][0], c[1] - p["center"][1]) <= rad + p["_r"] + 0.02 for p in obs):
            continue
        a, v = rng.uniform(-math.pi, math.pi), rng.uniform(0.0, 0.5)
        ob["velocity"] = (v * math.cos(a), v * math.sin(a))
        if reactive_every and len(obs) % reactive_every == 0:
            ob["velocity"] = (0.0, 0.0)
            ob["behavior"] = dict(name="rvo", vxmax=0.4, vymax=0.4, wander=True)
        ob["_r"] = rad
        obs.append(ob)
    for ob in obs:
        del ob["_r"]
    return obs


def test_no_moving_obstacle_ever_touches_another():
    """500 free-running oracle steps: two crowded 12 x 12 m scenes of 24 obstacles (one with a reactive obstacle in every three),
    a 40 x 40 m scene of 256 obstacles and a scene without contact.  After every step, no pair with a mover touches in a contact
    scene; the scene without contact has overlapping pairs."""
    rng = np.random.default_rng(4)
    scenes = []
    for b, (n, size, reactive) in enumerate(((24, 12.0, 0), (24, 12.0, 3), (256, 40.0, 0), (24, 12.0, 0))):
        sc = _scene(_crowded(rng, n, (0.0, 0.0, size, size), reactive), contact=b != 3)
        sc["bounds"] = (0.0, 0.0, size, size)
        scenes.append(sc)
    o = _oracle(scenes, seed=3)
    movers = o.moving()
    assert o.touching_pairs(movers) == []
    plain_overlaps = 0
    b3 = slice(o.obs_begin[3], o.obs_begin[4])
    for k in range(500):
        o.margins = o.rvo(np.zeros((4, 2)), envs=[1])
        o.move_all()
        assert o.touching_pairs(movers) == [], k
        if k % 50 == 0:
            plain_overlaps += sum(touches(o.shapes[i], tuple(o.obs[i, :2]), o.shapes[j], tuple(o.obs[j, :2]))
                                  for i in range(b3.start, b3.stop) for j in range(i + 1, b3.stop))
    assert o.obounces.sum() > 0 and sum(o.otaken.values()) == o.obounces.sum() and o.otaken["D"] > 0
    assert plain_overlaps > 0
