"""Actuation limits and noise of the batched world, on the CPU: the float64 restatement (tests/world_actuation_oracle.py) against
hand-computed limits, the independence and statistics of its noise streams, and the Python-side refusals of set_actuation and
set_lidar_noise."""
import math

import numpy as np
import pytest

from neupan_b200.robot import robot as Robot
from neupan_b200.world import ACTUATION_DEFAULTS, check_lidar_noise, pack_actuation
from oracle.world import draw_goal, rvo_key, splitmix64_at
from world_actuation_oracle import TAG_LIDAR, TAG_MOTION, Actuation, lidar_noise, limit, noise_key, normal, normals

INF = math.inf
DIFF = Robot(10, 0.1, kinematics="diff", length=1.6, width=2.0)
ACKER = Robot(10, 0.1, kinematics="acker", length=4.6, width=1.6, wheelbase=3)
OMNI = Robot(10, 0.1, kinematics="omni", vertices=[[-0.8, -1.0], [-1.8, 1.0], [1.8, 1.0], [0.8, -1.0]])


# (action, cmd_prev, (vel_min, vel_max, acce), dt) -> the limited command, computed by hand
LIMIT_TABLE = [
    ("rate limit only, rising", 2.0, 0.5, (-INF, INF, 1.0), 0.1, 0.6),
    ("rate limit only, falling", -2.0, 0.5, (-INF, INF, 1.0), 0.1, 0.4),
    ("rate limit only, inside", 0.55, 0.5, (-INF, INF, 1.0), 0.1, 0.55),
    ("bound only, above", 9.0, 0.0, (-8.0, 8.0, INF), 0.1, 8.0),
    ("bound only, below", -9.0, 0.0, (-8.0, 8.0, INF), 0.1, -8.0),
    ("both, the rate binds", 9.0, 7.5, (-8.0, 8.0, 4.0), 0.1, 7.9),
    ("both, the bound binds", 9.0, 7.9, (-8.0, 8.0, 4.0), 0.1, 8.0),
    ("a negative command", -3.0, -1.0, (-2.0, 2.0, 5.0), 0.1, -1.5),
    ("a negative command, bound", -3.0, -1.8, (-2.0, 2.0, 5.0), 0.1, -2.0),
    ("acker steering, bound", 1.2, 0.0, (-1.0, 1.0, INF), 0.1, 1.0),
    ("acker steering, rate", -0.9, 0.2, (-1.0, 1.0, 2.0), 0.1, 0.0),
    ("no limits: the action itself", -0.3, 5.0, (-INF, INF, INF), 0.1, -0.3),
]


@pytest.mark.parametrize("case", LIMIT_TABLE, ids=[c[0] for c in LIMIT_TABLE])
def test_limits_match_the_hand_computed_table(case):
    _, a, prev, row, dt, want = case
    assert limit(a, prev, row, dt) == pytest.approx(want, abs=1e-15)


def test_actuation_applies_per_component_and_per_type_and_keeps_cmd_prev():
    """Two types (diff with both limits, acker with a steering bound), a collided robot, and cmd_prev carried across steps."""
    rows = pack_actuation([dict(vel_min=(-1.0, -2.0), vel_max=(1.0, 2.0), acce=(2.0, 10.0)), dict(vel_min=(-8, -0.5), vel_max=(8, 0.5))],
                          [DIFF, ACKER])
    act = Actuation(rows, seed=0, N=3, dt=0.1)
    u = act.apply(np.float32([[3.0, -3.0], [0.5, 0.9], [1.0, 1.0]]), collided=[0, 0, 1], K=1, rtype=[0, 1, 0])
    assert np.allclose(u, [[0.2, -1.0], [0.5, 0.5], [0.0, 0.0]], atol=1e-15)
    assert np.array_equal(act.cmd, u)
    u = act.apply(np.float32([[3.0, -3.0], [0.5, -0.9], [1.0, 1.0]]), collided=[0, 0, 0], K=1, rtype=[0, 1, 0])
    assert np.allclose(u, [[0.4, -2.0], [0.5, -0.5], [0.2, 1.0]], atol=1e-15)
    act.apply(np.zeros((3, 2), np.float32), collided=[1, 0, 0], K=1, rtype=[0, 1, 0])
    assert (act.cmd[0] == 0.0).all()  # a collided robot's cmd_prev becomes 0


def test_defaults_leave_the_action_bit_for_bit():
    rows = pack_actuation([{}, {}, {}], [DIFF, ACKER, OMNI])
    assert np.array_equal(rows[0], [-INF, -INF, INF, INF, INF, INF, 0, 0, 0, 0])
    a = np.random.default_rng(1).normal(0, 3, (30, 2)).astype(np.float32)
    a[0] = (-0.0, 0.0)
    act = Actuation(rows, seed=4, N=30, dt=0.1)
    for n in range(3):
        u = act.apply(a, np.zeros(30, np.int32), K=3, rtype=np.arange(30) % 3, n=n)
        assert np.array_equal(u.view(np.int64), a.astype(np.float64).view(np.int64))


def test_stream_keys_are_independent():
    seed, e, k, n = 7, 3, 2, 11
    z0 = normal(noise_key(seed, TAG_MOTION, e, k, n), 1)
    for what, key in (("seed", (8, e, k, n)), ("e", (seed, 4, k, n)), ("k", (seed, e, 1, n)), ("n", (seed, e, k, 12))):
        assert normal(noise_key(key[0], TAG_MOTION, *key[1:]), 1) != z0, what
    assert normal(noise_key(seed, TAG_MOTION, e, k, n), 0) != z0  # j
    assert normal(noise_key(seed, TAG_LIDAR, e, k, n), 1) != z0  # the domain tag


def test_lidar_motion_and_goal_streams_never_coincide():
    """Every raw 64-bit output the three uses draw for seeds 0..2, environments 0..3, robots / obstacles 0..3, steps or draws 0..7 and
    components / beams 0..7: no value appears in two of them (nor twice in one)."""
    outs = {"motion": [], "lidar": [], "goal": []}
    for seed in range(3):
        for e in range(4):
            for k in range(4):
                g = rvo_key(seed, e, k)
                outs["goal"] += [int(splitmix64_at(g, m)) for m in range(2 * 8 * 8)]
                for n in range(8):
                    for tag, name in ((TAG_MOTION, "motion"), (TAG_LIDAR, "lidar")):
                        key = noise_key(seed, tag, e, k, n)
                        outs[name] += [int(splitmix64_at(key, m)) for m in range(16)]
    allv = [v for vs in outs.values() for v in vs]
    assert len(set(allv)) == len(allv)
    # the goal draws themselves are those of oracle.world.draw_goal (the rvo stream is unchanged)
    gx, _ = draw_goal(1, 2, 3, 0, (0.0, 0.0, 1.0, 1.0))
    assert gx == float(np.uint64(splitmix64_at(rvo_key(1, 2, 3), 0)) >> np.uint64(11)) * 2.0 ** -53


def test_a_million_draws_are_standard_normal():
    n = 10 ** 6
    z = normals(noise_key(2026, TAG_LIDAR, 5, 1, 9), np.arange(n))
    assert z[:50].tolist() == pytest.approx([normal(noise_key(2026, TAG_LIDAR, 5, 1, 9), j) for j in range(50)], rel=1e-14)
    assert abs(z.mean()) < 5.0 / math.sqrt(n)
    assert abs(z.var() - 1.0) < 0.01


def test_a_sub_range_of_environments_reproduces_the_full_batch():
    """Environment b's motion and lidar noise depend on (seed, b, k, n, j) only: environments 2..4 of a batch of 6 (K = 2), run
    alone with their own indices, draw the same."""
    B, K, R = 6, 2, 40
    rng = np.random.default_rng(3)
    rows = pack_actuation([dict(acce=(2.0, 3.0), alpha=(0.05, 0.01, 0.02, 0.04))], [DIFF])
    full, part = Actuation(rows, 9, B * K, 0.1), Actuation(rows, 9, 3 * K, 0.1)
    sub = slice(2 * K, 5 * K)
    for n in range(4):
        a = rng.uniform(-2, 2, (B * K, 2)).astype(np.float32)
        col = np.zeros(B * K, np.int32)
        uf = full.apply(a, col, K, n=n)
        up = part.apply(a[sub], col[sub], K, n=n, scene=[2, 3, 4])
        assert np.array_equal(uf[sub], up) and np.array_equal(full.cmd[sub], part.cmd)
        ranges = rng.uniform(0.5, 9.0, (B * K, R))
        hit = np.where(rng.uniform(size=(B * K, R)) < 0.7, 0, -1)
        rf = lidar_noise(ranges, hit, K, 5, 0.05, 0.0, 10.0, n=n)
        rp = lidar_noise(ranges[sub], hit[sub], K, 5, 0.05, 0.0, 10.0, n=n, envs=[2, 3, 4])
        assert np.array_equal(rf[sub], rp)
        assert np.array_equal(rf[hit < 0], ranges[hit < 0]) and not np.array_equal(rf[hit >= 0], ranges[hit >= 0])


def test_lidar_noise_clamps_to_the_range_limits():
    ranges = np.array([[0.01, 9.99, 5.0, 10.0]])
    hit = np.array([[0, 1, 2, -1]])
    out = lidar_noise(ranges, hit, 1, 0, 100.0, 0.1, 10.0)
    assert ((out[0, :3] == 0.1) | (out[0, :3] == 10.0)).all() and out[0, 3] == 10.0


BAD = [
    ("NaN", [dict(vel_max=(math.nan, 1.0))], [DIFF]),
    ("vel_min > vel_max", [dict(vel_min=(1.0, 0.0), vel_max=(0.5, 1.0))], [DIFF]),
    ("vel_min = inf", [dict(vel_min=(INF, 0.0))], [DIFF]),
    ("acce = 0", [dict(acce=(0.0, 1.0))], [DIFF]),
    ("acce < 0", [dict(acce=(1.0, -1.0))], [DIFF]),
    ("negative alpha", [dict(alpha=(0.0, -0.1, 0.0, 0.0))], [DIFF]),
    ("infinite alpha", [dict(alpha=(INF, 0.0, 0.0, 0.0))], [DIFF]),
    ("acker steering at pi/2", [{}, dict(vel_min=(-8.0, -math.pi / 2), vel_max=(8.0, 1.0))], [DIFF, ACKER]),
    ("acker steering above pi/2", [{}, dict(vel_max=(8.0, 2.0))], [DIFF, ACKER]),
    ("a dict per type", [{}], [DIFF, ACKER]),
    ("an unknown key", [dict(vmax=(1.0, 1.0))], [DIFF]),
    ("two values", [dict(alpha=(0.1, 0.1))], [DIFF]),
]


@pytest.mark.parametrize("case", BAD, ids=[c[0] for c in BAD])
def test_set_actuation_refusals_raise_value_error(case):
    _, limits, robots = case
    with pytest.raises(ValueError):
        pack_actuation(limits, robots)


def test_steering_limits_of_other_kinematics_and_unbounded_acker_are_accepted():
    rows = pack_actuation([dict(vel_min=(-8, -3.14), vel_max=(8, 3.14)), dict(vel_min=(-8, -1), vel_max=(8, 1)), {}], [DIFF, ACKER, OMNI])
    assert rows.shape == (3, 10) and set(ACTUATION_DEFAULTS) == {"vel_min", "vel_max", "acce", "alpha"}
    pack_actuation([{}, {}], [DIFF, ACKER])  # +-inf steering: no bound


@pytest.mark.parametrize("std,rmin", [(-0.1, 0.0), (math.nan, 0.0), (INF, 0.0), (0.1, -1.0), (0.1, 10.0), (0.1, math.nan)])
def test_set_lidar_noise_refusals_raise_value_error(std, rmin):
    with pytest.raises(ValueError):
        check_lidar_noise(std, rmin, 10.0)
    check_lidar_noise(0.0, 0.0, 10.0)
