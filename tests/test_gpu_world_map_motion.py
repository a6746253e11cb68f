"""Obstacles in occupancy maps on the GPU (nb_world_set_map_contact): flags that are all 0 equal a world without the call (bitwise,
the same launches); teacher-forced parity of obstacle rows, goals, draws and bounces against the float64 oracle
(tests/world_map_motion_oracle.py) for K = 1 diff, K = 4 acker and a mixed fleet with noise, maze and cave maps at 0.05 to 1 m;
an episode bank of rvo mazes with movers equals its plain run; closed-loop runs repeat bit for bit without a host synchronisation."""
import math

import numpy as np
import pytest
import torch

from gpu_helpers import record
from neupan_b200 import WorldBatch, _lib, rollout
from neupan_b200.world import maze, pack_behaviors, pack_fleet, pack_map_contact, pack_maps, pack_robot_types, pack_scenes_ex
from test_gpu_world import EXAMPLE_LIDAR, LIDAR, _oracle_cfg, _planner, _ulps
from test_gpu_world_fleet import _device
from test_gpu_world_map import _map_scenes
from test_gpu_world_mixed import _mixed_actions, _robot, _types_of
from world_map_motion_oracle import MapMotionOracleWorld

pytestmark = pytest.mark.gpu

DT = 0.1
LIDAR90 = dict(LIDAR, number=90)


def _outputs(w, act):
    a = [t for t in w.scan(hit=True) if torch.is_tensor(t)] + list(w.step(act))
    return a + [w.states, w.obstacles()] + list(w.flags())


def test_flags_all_zero_are_the_world_without_the_call():
    """maze movers with "blocks_obstacles" False (no call) and the same scenes with nb_world_set_map_contact of all-zero flags equal
    each other bit for bit over 30 steps, with the same launches; blocking the same scenes changes the obstacles' motion."""
    B = 64
    rb = _robot("diff")
    scenes = maze(B, seed=4, movers=8)
    for sc in scenes:
        sc["map"]["blocks_obstacles"] = False
    plain, zero = WorldBatch(B, rb, LIDAR90, DT), WorldBatch(B, rb, LIDAR90, DT)
    plain.set_scenes(scenes)
    zero.set_scenes(scenes)
    flags = np.zeros(B, np.int32)
    with torch.cuda.device(zero.device):
        _lib.check(_lib.load().nb_world_set_map_contact(zero._handle, B, flags.ctypes.data))
    lib = _lib.load()
    rng = np.random.default_rng(5)
    for _ in range(30):
        act = torch.from_numpy(np.column_stack([rng.uniform(-1, 2, B), rng.uniform(-0.5, 0.5, B)]).astype(np.float32)).cuda()
        outs, counts = [], []
        for w in (plain, zero):
            n0 = lib.nb_launch_count()
            outs.append(_outputs(w, act))
            counts.append(lib.nb_launch_count() - n0)
        assert counts == [2, 2]
        assert all(torch.equal(x, y) for x, y in zip(outs[0], outs[1]))
    plain.close(); zero.close()


def _blocking_scenes(B, K, seed, robots):
    """_map_scenes with the map blocking obstacles in 3 of every 4 mapped environments: there every moving obstacle is slowed to
    0.9 resolution / step_time (reactive: its vxmax, vymax) and the cells near its start are freed."""
    scenes = _map_scenes(B, K, seed, robots)
    for b, sc in enumerate(scenes):
        if "map" not in sc or b % 4 == 3:
            continue
        m = sc["map"]
        res, (x0, y0), occ = m["resolution"], m["origin"], m["occupancy"]
        H, W = occ.shape
        cx, cy = x0 + (np.arange(W) + 0.5) * res, y0 + (np.arange(H) + 0.5) * res
        top = 0.9 * res / DT
        for ob in sc["obstacles"]:
            beh = ob.get("behavior")
            v = np.asarray(ob.get("velocity", (0.0, 0.0)), np.float64)
            if beh and beh.get("name") == "rvo":
                s = min(1.0, top / math.hypot(beh["vxmax"], beh["vymax"]))
                beh["vxmax"], beh["vymax"] = beh["vxmax"] * s, beh["vymax"] * s
                if beh.get("speed") is not None:
                    beh["speed"] = min(beh["speed"], beh["vxmax"], beh["vymax"])
                beh["acce"] = min(beh.get("acce", 1.0), beh["vxmax"], beh["vymax"])
                beh["grid"] = min(beh.get("grid", 0.05), beh["vxmax"] / 4, beh["vymax"] / 4)
            elif not v.any():
                continue
            elif np.hypot(*v) > top:
                ob["velocity"] = tuple(v * (top / np.hypot(*v)))
            if "radius" in ob:
                rad = ob["radius"]
            else:
                rad = max(math.hypot(*p) for p in np.asarray(ob.get("vertices", ob.get("outline")), np.float64))
            d = np.hypot(cx[None, :] - ob["center"][0], cy[:, None] - ob["center"][1])
            occ[d <= rad + 1.5 * res] = False
        m["blocks_obstacles"] = True
    return scenes


RUNS = {"diff_K1": (("diff",), 1, 90), "acker_K4": (("acker",), 4, 37), "mixed3_K4": (("diff", "acker", "omni"), 4, 37)}


@pytest.mark.parametrize("run", list(RUNS))
def test_teacher_forced_map_contact_matches_the_oracle(run):
    """50 random-action steps of B = 128 scenes, most of whose maps block obstacles: before every step the oracle takes the
    device's state; obstacle rows, goals, draws and bounces must be bitwise equal, and hits, ranges, clearances, flags and states
    meet the map tests' bars.  Reactive obstacles keep the reactive tests' excuse (a robot decision margin below 1e-12)."""
    names, K, R = RUNS[run]
    B, steps, window = 128, 50, 1.5
    robots = [_robot(n) for n in names]
    kins = [r.kinematics for r in robots]
    lidar = dict(LIDAR, number=R, scan_offset=(0.1, 0.05, 0.1))
    scenes = _blocking_scenes(B, K, 31, robots)
    packed, beh, fleet, rtype = pack_scenes_ex(scenes), pack_behaviors(scenes), pack_fleet(scenes), pack_robot_types(scenes)
    w = WorldBatch(B, robots if len(robots) > 1 else robots[0], lidar, DT)
    w.set_scenes(scenes, seed=13, map_window=window)
    o = MapMotionOracleWorld(_oracle_cfg(robots[0], lidar), packed, beh, seed=13, fleet=fleet, K=K, types=_types_of(robots),
                             robot_type=rtype, maps=pack_maps(scenes), window=window, block=pack_map_contact(scenes))
    s0 = _device(w)
    assert np.array_equal(s0["goal"], o.goal) and np.array_equal(s0["draws"], o.draws)
    rng = np.random.default_rng(17)
    excused_obs, worst_state, wrong = 0, 0.0, []
    for k in range(steps):
        s = _device(w)
        o.obs[:], o.states[:], o.collided[:], o.arrived[:], o.goal[:], o.draws[:] = (s["obs"], s["states"], s["collided"], s["arrived"],
                                                                                     s["goal"], s["draws"])
        ranges, vel, _, hit = (t.cpu().numpy() if torch.is_tensor(t) else t for t in w.scan(hit=True))
        r64, v64, h64, _, _ = o.scan()
        assert np.array_equal(hit, h64), (k, np.argwhere(hit != h64)[:5])
        assert (_ulps(ranges, r64.astype(np.float32)) <= 1).all(), k
        assert np.array_equal(vel, v64.astype(np.float32)), k
        act = _mixed_actions(rng, kins, rtype, s["states"], K)
        margins = o.rvo(act)
        _, _, clear_o = o.step(act, rvo=False)
        col, arr, clear = (t.cpu().numpy() for t in w.step(torch.from_numpy(act).cuda()))
        d = _device(w)
        bounces = w.map_bounces().cpu().numpy()
        bad_env = set()
        for b in range(B):
            sl = slice(o.obs_begin[b], o.obs_begin[b + 1])
            bad = ~(np.all(d["obs"][sl] == o.obs[sl], 1) & np.all(d["goal"][sl] == o.goal[sl], 1) & (d["draws"][sl] == o.draws[sl])
                    & (bounces[sl] == o.bounces[sl]))
            for q in np.flatnonzero(bad) + sl.start:
                if margins[q] < 1e-12:
                    excused_obs += 1
                    bad_env.add(b)
                else:
                    wrong.append(("obstacle", k, b, int(q)))
        for b in bad_env:  # an excused environment restarts from the device's state (the oracle follows it)
            sl = slice(o.obs_begin[b], o.obs_begin[b + 1])
            o.bounces[sl] = bounces[sl]
        ok = np.ones(B * K, bool)
        for b in bad_env:
            ok[b * K:(b + 1) * K] = False
        worst_state = max(worst_state, float(np.abs(d["states"] - o.states)[ok].max()))
        assert np.array_equal(col[ok], o.collided[ok]) and np.array_equal(arr[ok], o.arrived[ok]), k
        u = _ulps(clear, clear_o.astype(np.float32))[ok]
        assert (u == 0).all(), (k, np.flatnonzero(u > 0)[:5])
    blocked = np.repeat(pack_map_contact(scenes), np.diff(o.obs_begin)).astype(bool)
    moving = (o.beh[:, 0] == 1.0) | np.any(o.obs[:, 2:4] != 0.0, 1)
    touching = sum(o.obstacle_touches_map(q) for q in np.flatnonzero(blocked & moving))
    record(f"world_map_motion_teacher_forced_{run}", envs=B, robots=B * K, steps=steps, blocking_envs=int(pack_map_contact(scenes).sum()),
           bounces=int(o.bounces.sum()), taken_B=o.taken["B"], taken_C=o.taken["C"], taken_D=o.taken["D"],
           rejected_draws=o.rejected_draws, draws=int(o.draws.sum()), excused_obstacles=excused_obs, max_state_err=worst_state,
           moving_touching_map=int(touching), mismatches=len(wrong))
    assert not wrong, wrong[:3]
    assert worst_state <= 1e-12
    assert touching == 0
    assert o.bounces.sum() > 0 and o.rejected_draws > 0  # OBSERVED: the counts per candidate are reported above
    w.close()


def test_episode_bank_of_rvo_mazes_with_movers_is_its_plain_run():
    """A bank of S = 12 maze(movers=8, behavior="rvo") scenes through 4 slots (at most 60 steps each), each scene driven by its own action table (row t of
    scene s at its step t): every scene's final robot state, flags, obstacle rows, goals, draws and bounces equal the plain run of
    the bank truncated at that scene's end step."""
    S, slots, T = 12, 4, 60
    rb = _robot("diff")
    scenes = maze(S, seed=6, movers=8, behavior="rvo", layouts=3)
    rng = np.random.default_rng(3)
    # forward speeds up to 3 m/s in a 5 m maze cell: most robots hit a wall, at different steps, so slots change scenes at different times
    table = np.stack([rng.uniform(0.0, 3.0, (S, T)), rng.uniform(-0.8, 0.8, (S, T))], -1).astype(np.float32)  # (S, T, 2)
    plain = WorldBatch(S, rb, LIDAR90, DT)
    plain.set_scenes(scenes, seed=9)
    hist = [(_device(plain), plain.map_bounces().cpu().numpy())]
    for t in range(T):
        plain.scan()
        plain.step(torch.from_numpy(table[:, t]).cuda())
        hist.append((_device(plain), plain.map_bounces().cpu().numpy()))
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
    obs, (goal, draws), bounces = ep.obstacles().cpu().numpy(), (x.cpu().numpy() for x in ep.goals()), ep.map_bounces().cpu().numpy()
    ob = pack_scenes_ex(scenes)[0]
    for s in range(S):
        h, hb = hist[end[s]]
        sl = slice(ob[s], ob[s + 1])
        assert np.array_equal(states[s], h["states"][s]) and col[s] == h["collided"][s] and arr[s] == h["arrived"][s], s
        assert np.array_equal(obs[sl], h["obs"][sl]) and np.array_equal(goal[sl], h["goal"][sl]) and np.array_equal(draws[sl], h["draws"][sl]), s
        assert np.array_equal(bounces[sl], hb[sl]), s
    record("world_map_motion_episodes", scenes=S, slots=slots, end_steps=end.tolist(), bounces=int(bounces.sum()), draws=int(draws.sum()))
    plain.close(); ep.close()


def test_closed_loop_runs_repeat_without_a_host_synchronisation():
    """Two identical closed-loop runs of C4's planner in maze(16, movers=8, behavior="rvo") give the same results, obstacle rows and
    bounces bit for bit, with the host never synchronised inside rollout."""
    B = 16
    scenes = maze(B, seed=2, movers=8, behavior="rvo")
    outs = []
    for _ in range(2):
        pl = _planner(B, EXAMPLE_LIDAR)
        pl.set_initial_paths([sc["path"] for sc in scenes])
        w = WorldBatch(B, pl.robot, EXAMPLE_LIDAR, pl.dt)
        w.set_scenes(scenes, seed=1)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = rollout(pl, w, 20)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        outs.append([out[k].cpu() for k in sorted(out)] + [w.obstacles().cpu(), w.map_bounces().cpu()])
        pl.close(); w.close()
    assert all(torch.equal(a, b) for a, b in zip(*outs))
