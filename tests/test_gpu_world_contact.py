"""Obstacle contact on the GPU (nb_world_set_obstacle_contact): a world without contact and one with all-zero flags equal a plain
world bit for bit with the same launches; teacher-forced parity of obstacle rows, goals, draws and both bounce counters against the
float64 oracle (tests/world_contact_oracle.py) for K = 1 diff, K = 4 acker and a mixed fleet, with and without blocking maps; hand-made
edge cases; free-running scenes in which no moving obstacle ever touches another; and an episode bank that equals its plain run."""
import math

import numpy as np
import pytest
import torch

from gpu_helpers import record
from neupan_b200 import WorldBatch, _lib
from neupan_b200.world import (EXAMPLE_RVO, dyna_non_obs, dyna_obs, pack_behaviors, pack_fleet, pack_map_contact, pack_maps,
                               pack_obstacle_contact, pack_robot_types, pack_scenes_ex, random_outline)
from test_gpu_world import LIDAR, _oracle_cfg, _ulps
from test_gpu_world_fleet import _device
from test_gpu_world_map_motion import _blocking_scenes
from test_gpu_world_mixed import _mixed_actions, _robot, _types_of
from world_contact_oracle import ContactOracleWorld

pytestmark = pytest.mark.gpu

DT = 0.1
LIDAR90 = dict(LIDAR, number=90)
SQUARE = [[-0.5, -0.5], [0.5, -0.5], [0.5, 0.5], [-0.5, 0.5]]
NOTCH = [[-2.0, -2.0], [2.0, -2.0], [2.0, 2.0], [0.5, 2.0], [0.5, -0.5], [-0.5, -0.5], [-0.5, 2.0], [-2.0, 2.0]]  # a U, open upwards


def _outputs(w, act):
    a = [t for t in w.scan(hit=True) if torch.is_tensor(t)] + list(w.step(act))
    return a + [w.states, w.obstacles()] + list(w.flags())


def _oracle(scenes, robots=None, lidar=LIDAR90, seed=0, K=1, window=1.0):
    robots = robots or [_robot("diff")]
    maps = pack_maps(scenes) if any("map" in sc for sc in scenes) else None
    return ContactOracleWorld(_oracle_cfg(robots[0], lidar), pack_scenes_ex(scenes), pack_behaviors(scenes), seed=seed, fleet=pack_fleet(scenes),
                              K=K, types=_types_of(robots), robot_type=pack_robot_types(scenes), maps=maps, window=window,
                              block=pack_map_contact(scenes) if maps is not None else None, contact=pack_obstacle_contact(scenes))


def _touching(o, rows):
    """Pairs with a mover that touch at the device's rows (the CPU predicate)."""
    movers = o.moving()
    o.obs[:] = rows
    return o.touching_pairs(movers)


def test_without_contact_or_with_zero_flags_the_world_is_unchanged():
    """dyna_obs without the key, the same scenes with nb_world_set_obstacle_contact of all-zero flags, and the same scenes after a
    contact run and a new set_scenes equal each other bit for bit over 50 steps, with the same launches (scan + step); a world with
    contact launches one more kernel per step; the call refuses a wrong B."""
    B = 64
    rb = _robot("diff")
    scenes = dyna_obs(B, seed=4)
    plain, zero, again = (WorldBatch(B, rb, LIDAR90, DT) for _ in range(3))
    plain.set_scenes(scenes)
    zero.set_scenes(scenes)
    lib = _lib.load()
    flags = np.zeros(B, np.int32)
    with torch.cuda.device(zero.device):
        assert lib.nb_world_set_obstacle_contact(zero._handle, B + 1, flags.ctypes.data) == _lib.NB_ERR_INVALID
        assert "B = 65 but the scenes were set for 64 environments" in lib.nb_last_error().decode()
        _lib.check(lib.nb_world_set_obstacle_contact(zero._handle, B, flags.ctypes.data))
    contact = dyna_obs(B, seed=4, contact=True)
    again.set_scenes(contact)
    rng = np.random.default_rng(5)
    for _ in range(10):
        act = torch.from_numpy(np.column_stack([rng.uniform(-1, 2, B), rng.uniform(-0.5, 0.5, B)]).astype(np.float32)).cuda()
        n0 = lib.nb_launch_count()
        _outputs(again, act)
        assert lib.nb_launch_count() - n0 == 3
    again.set_scenes(scenes)
    assert not again.obstacle_contact
    rng = np.random.default_rng(5)
    for _ in range(50):
        act = torch.from_numpy(np.column_stack([rng.uniform(-1, 2, B), rng.uniform(-0.5, 0.5, B)]).astype(np.float32)).cuda()
        outs, counts = [], []
        for w in (plain, zero, again):
            n0 = lib.nb_launch_count()
            outs.append(_outputs(w, act))
            counts.append(lib.nb_launch_count() - n0)
        assert counts == [2, 2, 2]
        assert all(torch.equal(x, y) and torch.equal(x, z) for x, y, z in zip(*outs))
    plain.close(); zero.close(); again.close()


def _contact_scenes(B, K, seed, robots):
    """_blocking_scenes (circles, polygons, outlines, about half reactive; maps in 7 of 8 environments, blocking in 3 of 4 of those)
    with obstacle contact in every environment but each eighth one.  An environment whose map does not block obstacles also gets
    a crowded cluster of 12 obstacles of the three kinds in a 7 x 7 m square, a third of them reactive.  In a contact environment a
    moving obstacle that starts touching an earlier one is dropped."""
    scenes = _blocking_scenes(B, K, seed, robots)
    for b, sc in enumerate(scenes):
        rng = np.random.default_rng([seed, b, 7])
        if not (sc.get("map") or {}).get("blocks_obstacles"):
            x0, y0, x1, y1 = sc["bounds"]
            cx, cy = rng.uniform(x0 + 4, x1 - 4), rng.uniform(y0 + 4, y1 - 4)
            for i in range(12):
                c = (float(cx + rng.uniform(-3.5, 3.5)), float(cy + rng.uniform(-3.5, 3.5)))
                ob = (dict(center=c, radius=float(rng.uniform(0.2, 0.5))), dict(center=c, vertices=SQUARE),
                      dict(center=c, outline=random_outline(rng, 0.5, 0.9, 0.5, int(rng.integers(4, 10)))))[i % 3]
                a = rng.uniform(-math.pi, math.pi)
                ob["velocity"] = (0.5 * math.cos(a), 0.5 * math.sin(a))
                if i % 3 == 1:
                    ob["velocity"] = (0.0, 0.0)
                    ob["behavior"] = dict(EXAMPLE_RVO)
                sc["obstacles"].append(ob)
        if b % 8 == 7:
            continue
        sc["obstacle_contact"] = True
        while True:  # drop the mover of the first touching pair until none is left
            o = _oracle([sc], robots, K=K)
            pairs = o.touching_pairs()
            if not pairs:
                break
            i, j = pairs[0]
            del sc["obstacles"][j if o.moving()[j] else i]
    return scenes


RUNS = {"diff_K1": (("diff",), 1, 90), "acker_K4": (("acker",), 4, 37), "mixed3_K4": (("diff", "acker", "omni"), 4, 37)}


@pytest.mark.parametrize("run", list(RUNS))
def test_teacher_forced_contact_matches_the_oracle(run):
    """50 random-action steps of B = 128 scenes: before every step the oracle takes the device's state; obstacle rows, goals, draws,
    map bounces and obstacle bounces must be bitwise equal, and hits, ranges, clearances, flags and states meet the map tests' bars.
    Reactive obstacles keep the reactive tests' excuse (a robot decision margin below 1e-12), which excuses their environment."""
    names, K, R = RUNS[run]
    B, steps, window = 128, 50, 1.5
    robots = [_robot(n) for n in names]
    kins = [r.kinematics for r in robots]
    lidar = dict(LIDAR, number=R, scan_offset=(0.1, 0.05, 0.1))
    scenes = _contact_scenes(B, K, 31, robots)
    w = WorldBatch(B, robots if len(robots) > 1 else robots[0], lidar, DT)
    w.set_scenes(scenes, seed=13, map_window=window)
    o = _oracle(scenes, robots, lidar, seed=13, K=K, window=window)
    s0 = _device(w)
    assert np.array_equal(s0["goal"], o.goal) and np.array_equal(s0["draws"], o.draws)
    rng = np.random.default_rng(17)
    excused_envs, worst_state, wrong = 0, 0.0, []
    for k in range(steps):
        s = _device(w)
        o.obs[:], o.states[:], o.collided[:], o.arrived[:], o.goal[:], o.draws[:] = (s["obs"], s["states"], s["collided"], s["arrived"],
                                                                                     s["goal"], s["draws"])
        ranges, vel, _, hit = (t.cpu().numpy() if torch.is_tensor(t) else t for t in w.scan(hit=True))
        r64, v64, h64, _, _ = o.scan()
        assert np.array_equal(hit, h64), (k, np.argwhere(hit != h64)[:5])
        assert (_ulps(ranges, r64.astype(np.float32)) <= 1).all(), k
        assert np.array_equal(vel, v64.astype(np.float32)), k
        act = _mixed_actions(rng, kins, pack_robot_types(scenes), s["states"], K)
        margins = o.rvo(act)
        _, _, clear_o = o.step(act, rvo=False)
        col, arr, clear = (t.cpu().numpy() for t in w.step(torch.from_numpy(act).cuda()))
        d = _device(w)
        mb, ob = w.map_bounces().cpu().numpy(), w.obstacle_bounces().cpu().numpy()
        bad_env = set()
        for b in range(B):
            sl = slice(o.obs_begin[b], o.obs_begin[b + 1])
            bad = ~(np.all(d["obs"][sl] == o.obs[sl], 1) & np.all(d["goal"][sl] == o.goal[sl], 1) & (d["draws"][sl] == o.draws[sl])
                    & (mb[sl] == o.bounces[sl]) & (ob[sl] == o.obounces[sl]))
            if bad.any():
                if (margins[sl] < 1e-12).any():
                    bad_env.add(b)
                else:
                    wrong.append(("obstacle", k, b, (np.flatnonzero(bad) + sl.start).tolist()))
        for b in bad_env:  # an excused environment restarts from the device's state (the oracle follows it)
            sl = slice(o.obs_begin[b], o.obs_begin[b + 1])
            o.obs[sl], o.bounces[sl], o.obounces[sl] = d["obs"][sl], mb[sl], ob[sl]
        excused_envs += len(bad_env)
        ok = np.ones(B * K, bool)
        for b in bad_env:
            ok[b * K:(b + 1) * K] = False
        worst_state = max(worst_state, float(np.abs(d["states"] - o.states)[ok].max()))
        assert np.array_equal(col[ok], o.collided[ok]) and np.array_equal(arr[ok], o.arrived[ok]), k
        u = _ulps(clear, clear_o.astype(np.float32))[ok]
        assert (u == 0).all(), (k, np.flatnonzero(u > 0)[:5])
    touching = o.touching_pairs()
    record(f"world_contact_teacher_forced_{run}", envs=B, robots=B * K, steps=steps, contact_envs=int(pack_obstacle_contact(scenes).sum()),
           obstacles=len(o.obs), obstacle_bounces=int(o.obounces.sum()), map_bounces=int(o.bounces.sum()), taken_B=o.otaken["B"],
           taken_C=o.otaken["C"], taken_D=o.otaken["D"], excused_envs=excused_envs, max_state_err=worst_state, touching=len(touching),
           mismatches=len(wrong))
    assert not wrong, wrong[:3]
    assert worst_state <= 1e-12
    assert touching == []
    assert o.obounces.sum() > 0 and o.otaken["D"] > 0
    w.close()


def _edge_scenes():
    far = dict(start=(1.0, 1.0, 0.0), goal=(1.5, 1.0), goal_threshold=0.1, path=None, bounds=(0.0, 0.0, 20.0, 20.0), obstacle_contact=True)
    dart = [[0.0, -1.2], [0.8, 0.2], [0.0, -0.2], [-0.8, 0.2]]  # a concave arrowhead pointing down
    return [
        dict(far, obstacles=[dict(center=(8.95, 10.0), radius=0.5, velocity=(0.5, 0.0)), dict(center=(11.05, 10.0), radius=0.5, velocity=(-0.5, 0.0))]),
        dict(far, obstacles=[dict(center=(10.0, 10.0), radius=0.5, velocity=(0.3, 0.3))]
             + [dict(center=(10.0 + dx, 10.0 + dy), radius=0.5) for dx, dy in ((1.02, 0.0), (-1.02, 0.0), (0.0, 1.02), (0.0, -1.02))]),
        dict(far, obstacles=[dict(center=(19.98, 10.0), radius=0.3, velocity=(0.5, 0.0)), dict(center=(19.25, 10.0), radius=0.425)]),
        dict(far, obstacles=[dict(center=(10.0, 10.0), outline=NOTCH), dict(center=(10.0, 13.0), radius=0.3, velocity=(0.0, -0.5))]),
        dict(far, obstacles=[dict(center=(10.0, 10.0), outline=NOTCH), dict(center=(10.0, 13.0), outline=dart, velocity=(0.0, -0.5))]),
    ]


def test_edge_cases_match_the_oracle():
    """Two circles head-on; a circle pinned between four static ones (D every step); a mirror at the rectangle into a neighbour (C);
    a circle entering an outline's notch without touching its walls, then stopped by its floor; an arrowhead outline whose shoulder
    vertices come down on the notch's arms.  80 free-running steps on the device and on the oracle: rows and bounces bitwise equal
    at every step."""
    scenes = _edge_scenes()
    B = len(scenes)
    w = WorldBatch(B, _robot("diff"), LIDAR90, DT)
    w.set_scenes(scenes)
    o = _oracle(scenes)
    act = np.zeros((B, 2), np.float32)
    for k in range(80):
        w.step(torch.from_numpy(act).cuda())
        o.move_all()
        assert np.array_equal(w.obstacles().cpu().numpy(), o.obs), k
        assert np.array_equal(w.obstacle_bounces().cpu().numpy(), o.obounces), k
        assert o.touching_pairs() == [], k
    ob = o.obounces
    b = o.obs_begin
    assert ob[b[0]] > 0 and ob[b[0] + 1] > 0                           # head-on
    assert ob[b[1]] == 80 and tuple(o.obs[b[1], :2]) == (10.0, 10.0)   # pinned: D every step
    assert ob[b[2]] > 0                                                # the mirror into the neighbour
    assert ob[b[3] + 1] > 0                                            # stopped by the notch's floor, never by its walls
    assert ob[b[4] + 1] > 0                                            # the arrowhead stopped on the notch's corner
    record("world_contact_edge_cases", bounces=ob.tolist(), taken=o.otaken)
    w.close()


@pytest.mark.parametrize("which", ["dyna_obs", "dyna_non_obs_rvo"])
def test_free_running_obstacles_never_touch(which):
    """200 steps of dyna_obs(contact=True) and dyna_non_obs(contact=True, behavior="rvo") with random actions: every 10 steps the
    obstacle rows are read back and checked with the CPU predicate, and no pair with a mover touches."""
    B = 128
    scenes = dyna_obs(B, seed=8, contact=True) if which == "dyna_obs" else dyna_non_obs(B, seed=8, behavior="rvo", contact=True)
    w = WorldBatch(B, _robot("diff"), LIDAR90, DT)
    w.set_scenes(scenes, seed=2)
    o = _oracle(scenes)
    rng = np.random.default_rng(1)
    checked = 0
    for k in range(200):
        act = torch.from_numpy(np.column_stack([rng.uniform(-1, 2, B), rng.uniform(-0.5, 0.5, B)]).astype(np.float32)).cuda()
        w.scan()
        w.step(act)
        if k % 10 == 9:
            assert _touching(o, w.obstacles().cpu().numpy()) == [], k
            checked += 1
    bounces = int(w.obstacle_bounces().sum().item())
    record(f"world_contact_free_running_{which}", envs=B, steps=200, checks=checked, obstacle_bounces=bounces)
    assert bounces > 0
    w.close()


def test_episode_bank_with_contact_is_its_plain_run():
    """A bank of S = 12 dyna_obs(contact=True, behavior="rvo") scenes through 4 slots (at most 60 steps each), each scene driven by
    its own action table: every scene's final robot state, flags, obstacle rows, goals, draws and obstacle bounces equal the plain
    run of the bank truncated at that scene's end step."""
    S, slots, T = 12, 4, 60
    rb = _robot("diff")
    scenes = dyna_obs(S, seed=6, behavior="rvo", contact=True)
    rng = np.random.default_rng(3)
    table = np.stack([rng.uniform(0.0, 3.0, (S, T)), rng.uniform(-0.8, 0.8, (S, T))], -1).astype(np.float32)  # (S, T, 2)
    plain = WorldBatch(S, rb, LIDAR90, DT)
    plain.set_scenes(scenes, seed=9)
    hist = [(_device(plain), plain.obstacle_bounces().cpu().numpy())]
    for t in range(T):
        plain.scan()
        plain.step(torch.from_numpy(table[:, t]).cuda())
        hist.append((_device(plain), plain.obstacle_bounces().cpu().numpy()))
    ep = WorldBatch(S, rb, LIDAR90, DT)
    ep.set_episodes(scenes, slots, T, seed=9)
    tstep = np.zeros(slots, np.int64)
    for _ in range(S * T):
        scene_of, reset = (x.cpu().numpy() for x in ep.slot_scenes())
        tstep[reset != 0] = 0
        act = np.stack([table[s, min(t, T - 1)] for s, t in zip(scene_of, tstep)])
        ep.scan()
        ep.step(torch.from_numpy(act).cuda())
        tstep += 1
        if int(ep.finished().item()) >= S:
            break
    res = ep.episodes()
    end = res["end_step"].cpu().numpy()
    assert (end > 0).all() and len(set(end.tolist())) > 1
    states, col, arr = (x.cpu().numpy() for x in ep.scene_states())
    obs, (goal, draws), bounces = ep.obstacles().cpu().numpy(), (x.cpu().numpy() for x in ep.goals()), ep.obstacle_bounces().cpu().numpy()
    ob = pack_scenes_ex(scenes)[0]
    for s in range(S):
        h, hb = hist[end[s]]
        sl = slice(ob[s], ob[s + 1])
        assert np.array_equal(states[s], h["states"][s]) and col[s] == h["collided"][s] and arr[s] == h["arrived"][s], s
        assert np.array_equal(obs[sl], h["obs"][sl]) and np.array_equal(goal[sl], h["goal"][sl]) and np.array_equal(draws[sl], h["draws"][sl]), s
        assert np.array_equal(bounces[sl], hb[sl]), s
    record("world_contact_episodes", scenes=S, slots=slots, end_steps=end.tolist(), bounces=int(bounces.sum()))
    plain.close(); ep.close()
