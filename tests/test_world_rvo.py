"""Reactive obstacles (behaviour kind 1) of the batched world, on the CPU: host validation through nb_world_check_behaviors, the
SplitMix64 goal draws, the trig-free cones of oracle/world.py against IR-SIM's atan2 / asin construction, hand-built
choices of the oracle, pack_behaviors and the scene builders (no device needed)."""
import ctypes as C
import hashlib
import math

import numpy as np
import pytest

from neupan_b200 import _lib, build as nb_build
from neupan_b200.robot import robot as Robot
from neupan_b200.world import EXAMPLE_RVO, dyna_non_obs, dyna_obs, make_config, pack_behaviors, pack_scenes_ex
from oracle.world import OracleWorld, cone, cone_trig, cross, draw_goal, inside_cone, splitmix64_at, u01

LIDAR = dict(angle_min=-math.pi, angle_max=math.pi, range_min=0.0, range_max=10.0, number=36)


@pytest.fixture(scope="module")
def lib():
    nb_build.build()
    return _lib.load()


def _rvo(**kw):
    return dict(dict(name="rvo", vxmax=0.5, vymax=0.5), **kw)


def _scene(obstacles, bounds=(-10.0, -10.0, 10.0, 10.0), start=(-8.0, -8.0, 0.0)):
    return dict(obstacles=obstacles, bounds=bounds, start=start, goal=(8.0, 8.0), goal_threshold=0.3)


def _cfg(kin="diff"):
    rb = Robot(10, 0.1, kinematics=kin, length=1.6, width=2.0)
    return dict(kinematics=kin, step_time=0.1, wheelbase=rb.L, angle_min=LIDAR["angle_min"], angle_max=LIDAR["angle_max"],
                range_max=LIDAR["range_max"], number=LIDAR["number"], scan_offset=(0.0, 0.0, 0.0),
                robot_vertices=np.asarray(rb.vertices, np.float64).T), rb


# ---- host validation ---------------------------------------------------------------------------------------------------------

def _check(lib, cfg, scenes, beh=None, seed=0):
    packed = pack_scenes_ex(scenes)
    beh = pack_behaviors(scenes) if beh is None else beh
    return lib.nb_world_check_behaviors(C.byref(cfg), len(scenes), *[C.c_void_p(a.ctypes.data) for a in packed], C.c_void_p(beh.ctypes.data),
                                        C.c_uint64(seed))


def test_host_validation_of_behaviours(lib):
    rb = Robot(10, 0.1, kinematics="diff", length=1.6, width=2.0)
    cfg = make_config(rb, LIDAR, 0.1, max_envs=4)
    const = dict(center=(0.0, 0.0), radius=0.5, velocity=(0.1, 0.0))

    def scenes(**kw):
        ob = dict(center=kw.pop("center", (3.0, 0.0)), radius=0.5, behavior=_rvo(**kw))
        return [_scene([const, ob])]

    assert _check(lib, cfg, scenes()) == _lib.NB_OK
    assert _check(lib, cfg, scenes(goal=(9.0, -9.0), wander=True)) == _lib.NB_OK
    assert _check(lib, cfg, scenes(grid=1.0 / 64, acce=0.5)) == _lib.NB_OK  # exactly 64 candidates per axis
    beh = pack_behaviors(scenes())
    beh[0, 1:] = np.nan  # a kind-0 row is not read
    assert _check(lib, cfg, scenes(), beh) == _lib.NB_OK
    refusals = [
        (dict(), (0, 2.0), "obstacle 1 has behaviour kind 2"),
        (dict(), (4, math.nan), "obstacle 1: behaviour column 4 is not finite"),
        (dict(), (12, math.inf), "obstacle 1: behaviour column 12 is not finite"),
        (dict(), (7, 1.0), "obstacle 1: the goal must be finite, or NaN in both"),  # goal y stays NaN
        (dict(goal=(1.0, math.inf)), None, "obstacle 1: the goal must be finite"),
        (dict(vxmax=0.0), None, "obstacle 1: vxmax must be positive"),
        (dict(vymax=-1.0), None, "obstacle 1: vymax must be positive"),
        (dict(acce=0.0), None, "obstacle 1: acce must be positive"),
        (dict(factor=0.0), None, "obstacle 1: factor must be positive"),
        (dict(speed=0.0), None, "obstacle 1: speed must be positive"),
        (dict(goal_threshold=0.0), None, "obstacle 1: goal_threshold must be positive"),
        (dict(neighbor_range=0.0), None, "obstacle 1: neighbor_range must be positive"),
        (dict(grid=0.0), None, "obstacle 1: grid must be positive"),
        (dict(min_speed=-0.1), None, "obstacle 1: min_speed must be >= 0"),
        (dict(), (6, 0.5), "obstacle 1: wander must be 0 or 1"),
        (dict(grid=0.01), None, "obstacle 1: up to 100 candidate velocities on an axis (at most 64)"),
        (dict(grid=1.0 / 64, acce=0.6, vxmax=0.5 + 1.0 / 128), None, "obstacle 1: up to 65 candidate velocities on an axis (at most 64)"),
        (dict(center=(10.5, 0.0)), None, "obstacle 1 is reactive but its centre starts outside the rectangle of environment 0"),
        (dict(vymax=200.0, acce=0.01), None, "obstacle 1: vymax * step_time exceeds the rectangle of environment 0"),
        (dict(goal=(0.0, 10.5)), None, "obstacle 1: its goal lies outside the rectangle of environment 0"),
    ]
    for kw, poke, text in refusals:
        sc = scenes(**kw)
        beh = pack_behaviors(sc)
        if poke:
            beh[1, poke[0]] = poke[1]
        assert _check(lib, cfg, sc, beh) == _lib.NB_ERR_INVALID, text
        assert text in lib.nb_last_error().decode(), (text, lib.nb_last_error().decode())
    # the scenes are checked first, with their own messages
    bad = [_scene([dict(center=(0.0, 0.0), radius=-1.0), dict(center=(3.0, 0.0), radius=0.5, behavior=_rvo())])]
    assert _check(lib, cfg, bad) == _lib.NB_ERR_INVALID and "positive radius" in lib.nb_last_error().decode()
    assert lib.nb_world_check_behaviors(C.byref(cfg), 1, *[C.c_void_p(a.ctypes.data) for a in pack_scenes_ex(scenes())], None, 0) == _lib.NB_ERR_INVALID
    assert "null behaviors" in lib.nb_last_error().decode()


def test_pack_behaviors():
    sc = [_scene([dict(center=(0.0, 0.0), radius=0.5), dict(center=(1.0, 0.0), radius=0.5, behavior={"name": "constant"}),
                  dict(center=(2.0, 0.0), radius=0.5, behavior=_rvo(vymax=0.4, wander=True, goal=(1.0, 2.0)))]),
          _scene([dict(center=(3.0, 0.0), vertices=[[0, 0], [1, 0], [0, 1]], behavior=_rvo())])]
    beh = pack_behaviors(sc)
    assert beh.shape == (4, 13) and beh.dtype == np.float64 and not beh[:2].any()
    assert beh[2].tolist() == [1.0, 0.5, 0.4, 1.0, 1.0, 0.4, 1.0, 1.0, 2.0, 0.3, 10.0, 0.05, 0.3]
    assert beh[3, 0] == 1.0 and beh[3, 6] == 0.0 and np.isnan(beh[3, 7:9]).all()
    for b in ({"name": "orca"}, {"name": "rvo", "vxmax": 0.5}, _rvo(speeed=1.0)):
        with pytest.raises(ValueError):
            pack_behaviors([_scene([dict(center=(0.0, 0.0), radius=0.5, behavior=b)])])


# ---- generator ---------------------------------------------------------------------------------------------------------------

def test_splitmix64_matches_the_published_values():
    # the reference splitmix64.c outputs for the seeds 1234567 and 1477776061723855037
    assert [int(splitmix64_at(1234567, n)) for n in range(5)] == [6457827717110365317, 3203168211198807973, 9817491932198370423,
                                                                   4593380528125082431, 16408922859458223821]
    assert [int(splitmix64_at(1477776061723855037, n)) for n in range(3)] == [1985237415132408290, 2979275885539914483,
                                                                               13511426838097143398]
    assert u01(0) == 0.0 and u01(2 ** 64 - 1) == 1.0 - 2.0 ** -53


def test_goal_draws_lie_in_the_rectangle_and_differ_per_stream():
    bounds = (-3.0, 2.0, 5.0, 4.0)
    goals = np.array([draw_goal(seed, b, i, n, bounds) for seed in (0, 1) for b in range(4) for i in range(4) for n in range(8)])
    assert (goals[:, 0] >= -3.0).all() and (goals[:, 0] < 5.0).all() and (goals[:, 1] >= 2.0).all() and (goals[:, 1] < 4.0).all()
    assert len(np.unique(goals, axis=0)) == len(goals)
    assert draw_goal(7, 3, 2, 5, bounds) == draw_goal(7, 3, 2, 5, bounds)


# ---- oracle --------------------------------------------------------------------------------------------------------------------

def test_trig_free_cones_agree_with_the_atan2_asin_construction():
    """10^4 random cones and candidates: the inside decision of the trig-free cone equals IR-SIM's, except for candidates within
    1e-9 of a cone edge."""
    rng = np.random.default_rng(11)
    near, on_edge, n_in, n = 0, 0, 0, 10_000
    for _ in range(n):
        ci, cj = rng.uniform(-5, 5, 2), rng.uniform(-5, 5, 2)
        if rng.uniform() < 0.1:  # overlapping circles: D' = R
            cj = ci + rng.normal(0, 0.3, 2)
        vi, vj = rng.uniform(-1, 1, 2), rng.uniform(-1, 1, 2)
        ri, rj = rng.uniform(0.1, 1.5, 2)
        a, t = cone(ci, vi, ri, cj, vj, rj), cone_trig(ci, vi, ri, cj, vj, rj)
        for _ in range(4):
            v = rng.uniform(-1.5, 1.5, 2)
            if rng.uniform() < 0.05:  # a candidate on an edge of the cone (up to rounding)
                d = a[1] if rng.uniform() < 0.5 else a[2]
                s = rng.uniform(0.1, 2.0)
                v = np.array([a[0][0] + s * d[0], a[0][1] + s * d[1]])
                on_edge += 1
            n_in += inside_cone(a, *v)
            if inside_cone(a, *v) != inside_cone(t, *v):
                wx, wy = v[0] - a[0][0], v[1] - a[0][1]
                edge = min(abs(cross(a[1], wx, wy)), abs(cross(a[2], wx, wy)))
                assert edge < 1e-9, (ci, cj, vi, vj, ri, rj, v)
                near += 1
    print(f"OBSERVED trig-free vs atan2/asin cones: {near} of {4 * n} decisions differ ({on_edge} candidates were placed on an edge), "
          f"all within 1e-9 of an edge; {n_in} inside")
    assert near <= on_edge and 0.1 * 4 * n < n_in < 0.9 * 4 * n


def _oracle(scenes, seed=0, kin="diff"):
    cfg, _ = _cfg(kin)
    return OracleWorld(cfg, pack_scenes_ex(scenes), pack_behaviors(scenes), seed)


def test_a_free_obstacle_heads_for_its_goal():
    o = _oracle([_scene([dict(center=(0.0, 0.0), radius=0.5, behavior=_rvo(goal=(5.0, 0.0)))])])
    o.step(np.zeros((1, 2), np.float32))
    # the window [-0.5, 0.5) in steps of 0.05 from rest: the closest candidate to (0.5, 0) is lo + 19 grid
    assert tuple(o.obs[0, 2:4]) == (-0.5 + 19 * 0.05, 0.0) and o.obs[0, 0] == (-0.5 + 19 * 0.05) * 0.1
    o = _oracle([_scene([dict(center=(0.0, 0.0), radius=0.5, behavior=_rvo(goal=(5.0, 5.0)))])])
    o.step(np.zeros((1, 2), np.float32))
    vx, vy = o.obs[0, 2:4]
    assert abs(vx - vy) < 1e-12 and abs(math.hypot(vx, vy) - 0.5) < 0.05  # the grid point closest to 0.5 (cos 45, sin 45)


def test_a_head_on_neighbour_turns_the_obstacle_and_an_arrival_draws_or_parks():
    sc = [_scene([dict(center=(0.0, 0.0), radius=0.5, behavior=_rvo(goal=(5.0, 0.0))),
                  dict(center=(2.0, 0.0), radius=0.5, velocity=(-0.5, 0.0))])]
    o = _oracle(sc)
    o.step(np.zeros((1, 2), np.float32))
    vx, vy = o.obs[0, 2:4]
    assert vy != 0.0 and math.hypot(vx, vy) >= 0.3
    # arrival: wander draws goal 1 of the stream, no wander parks
    for wander in (True, False):
        o = _oracle([_scene([dict(center=(1.0, 1.0), radius=0.5, velocity=(0.2, 0.0), behavior=_rvo(goal=(1.1, 1.0), wander=wander))])], seed=5)
        o.step(np.zeros((1, 2), np.float32))
        if wander:
            assert tuple(o.goal[0]) == draw_goal(5, 0, 0, 0, (-10.0, -10.0, 10.0, 10.0)) and o.draws[0] == 1
        else:
            assert tuple(o.obs[0, 2:4]) == (0.0, 0.0) and tuple(o.goal[0]) == (1.1, 1.0) and o.draws[0] == 0
    o = _oracle([_scene([dict(center=(1.0, 1.0), radius=0.5, behavior=_rvo())])], seed=9)
    assert tuple(o.goal[0]) == draw_goal(9, 0, 0, 0, (-10.0, -10.0, 10.0, 10.0)) and o.draws[0] == 1


# ---- scene builders ----------------------------------------------------------------------------------------------------------

def _digest(scenes):
    h = hashlib.sha256()
    for a in pack_scenes_ex(scenes):
        h.update(np.ascontiguousarray(a).tobytes())
    for s in scenes:
        h.update(np.ascontiguousarray(s["path"]).tobytes())
    return h.hexdigest()


# pack_scenes_ex + paths of builder(16, seed=3) before the builders took a behaviour
DIGESTS = {"dyna_obs": "f1bdb17e794a1f144b329aba541fedb12406dcbbe2bc9585a4008841c262754c",
           "dyna_non_obs": "7f38b6e32a26f9856d5baded60c2610a5fe38718f0db78204ca36d1eb2e57025"}


@pytest.mark.parametrize("builder", [dyna_obs, dyna_non_obs])
def test_scene_builders_keep_their_default_output_and_add_the_examples_behaviour(lib, builder):
    assert _digest(builder(16, seed=3)) == DIGESTS[builder.__name__]
    assert _digest(builder(16, seed=3, behavior="constant")) == DIGESTS[builder.__name__]
    const, rvo = builder(16, seed=3), builder(16, seed=3, behavior="rvo")
    pc, pr = pack_scenes_ex(const), pack_scenes_ex(rvo)
    for k in (0, 2, 3, 4, 5):
        assert np.array_equal(pc[k], pr[k])
    assert np.array_equal(pc[1][:, [0, 1, 4]], pr[1][:, [0, 1, 4]]) and not pr[1][:, 2:4].any()
    beh = pack_behaviors(rvo)
    assert (beh[:, 0] == 1.0).all() and (beh[:, 1:3] == 0.5).all() and (beh[:, 6] == 1.0).all() and (beh[:, 9] == 0.3).all()
    assert all(ob["behavior"] == EXAMPLE_RVO for sc in rvo for ob in sc["obstacles"])
    rb = Robot(10, 0.1, kinematics="diff", length=1.6, width=2.0)
    assert _check(lib, make_config(rb, LIDAR, 0.1, max_envs=16), rvo) == _lib.NB_OK
    with pytest.raises(ValueError):
        builder(2, behavior="orca")
