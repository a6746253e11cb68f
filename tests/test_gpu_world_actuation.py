"""Actuation limits and noise of the batched world on the GPU (nb_world_set_actuation, nb_world_set_lidar_noise): defaults equal a
world without them bit for bit; teacher-forced parity with the float64 restatement (tests/world_actuation_oracle.py over the world
oracles) for limits alone, for limits with motion and lidar noise, and with obstacle contact and blocking maps; reproducibility
from the seeds and independence of B; and an episode bank with noise that equals the plain run of each scene."""
import math

import numpy as np
import pytest
import torch

from gpu_helpers import record
from neupan_b200 import WorldBatch
from neupan_b200.world import dyna_obs, maze, mixed_swap, pack_actuation, pack_robot_types
from test_gpu_world import LIDAR, _ulps
from test_gpu_world_contact import _contact_scenes, _oracle
from test_gpu_world_mixed import _robot
from world_actuation_oracle import Actuation, lidar_noise

pytestmark = pytest.mark.gpu

DT = 0.1
LIMITS = {  # per kinematics: bounds and rate limits that bind for the random actions below
    "diff": dict(vel_min=(-1.0, -1.0), vel_max=(1.5, 1.0), acce=(2.0, 3.0)),
    "acker": dict(vel_min=(-1.0, -0.6), vel_max=(2.0, 0.6), acce=(3.0, 2.0)),
    "omni": dict(vel_min=(-1.0, -1.0), vel_max=(1.0, 1.0), acce=(1.5, 1.5)),
}
ALPHA = (0.03, 0.02, 0.01, 0.03)


def _device(w):
    c, a = w.flags()
    return dict(obs=w.obstacles().cpu().numpy(), states=w.states.cpu().numpy(), collided=c.cpu().numpy(), arrived=a.cpu().numpy(),
                cmd=w.commands().cpu().numpy())


def _actions(rng, n):
    return np.column_stack([rng.uniform(-3, 3, n), rng.uniform(-1.5, 1.5, n)]).astype(np.float32)


def _outputs(w, act):
    out = [t for t in w.scan(hit=True) if torch.is_tensor(t)] + list(w.step(act))
    return out + [w.states, w.obstacles(), w.commands()] + list(w.flags())


@pytest.mark.parametrize("scene", ["dyna_obs", "maze_movers"])
def test_defaults_are_bitwise_a_world_without_them(scene):
    """set_actuation with every key at its default and range_std = 0 leave scans, steps, states, obstacles and flags bit for bit those
    of a world that never called them, over 50 steps; cmd_prev is the action itself there."""
    B = 64
    rb = _robot("diff")
    lidar = dict(LIDAR, number=90)
    scenes = dyna_obs(B, seed=3) if scene == "dyna_obs" else maze(B, seed=3, layouts=8, movers=8)
    ws = [WorldBatch(B, rb, lidar, DT) for _ in range(2)]
    for w in ws:
        w.set_scenes(scenes)
    ws[1].set_actuation([{}])
    ws[1].set_lidar_noise(0.0, seed=5)
    rng = np.random.default_rng(2)
    for k in range(50):
        act = torch.from_numpy(_actions(rng, B)).cuda()
        frozen = ws[1].flags()[0].bool()[:, None]
        a, b = _outputs(ws[0], act), _outputs(ws[1], act)
        for i, (x, y) in enumerate(zip(a, b)):
            if i != 8:  # 8: the commands
                assert torch.equal(x, y), (k, i)
        # cmd_prev: zeros without set_actuation; with the defaults the action itself, 0 for a robot that had collided
        assert (a[8] == 0).all() and torch.equal(b[8], torch.where(frozen, 0.0, act.double())), k
    for w in ws:
        w.close()


def _teacher_forced(w, o, A, scenes, K, steps, seed, noise, rng):
    """Before every step the oracle takes the device's state and cmd_prev; the scan (with lidar noise), cmd_prev (bitwise), flags,
    states and clearances must agree.  Reactive obstacles keep the reactive tests' excuse (a decision margin below 1e-12)."""
    std, rmin, rmax = noise
    rtype = pack_robot_types(scenes)
    B = len(scenes)
    worst, excused, ulp1 = 0.0, 0, 0
    for k in range(steps):
        s = _device(w)
        o.obs[:], o.states[:], o.collided[:], o.arrived[:] = s["obs"], s["states"], s["collided"], s["arrived"]
        A.cmd[:] = s["cmd"]
        ranges, vel, _, hit = (t.cpu().numpy() if torch.is_tensor(t) else t for t in w.scan(hit=True))
        r64, v64, h64, _, _ = o.scan()
        assert np.array_equal(hit, h64), (k, np.argwhere(hit != h64)[:5])
        r64 = lidar_noise(r64, h64, K, seed, std, rmin, rmax, n=k) if std > 0 else r64
        assert (_ulps(ranges, r64.astype(np.float32)) <= 1).all(), k
        assert np.allclose(vel, v64, rtol=1e-6, atol=0), k
        act = _actions(rng, B * K)
        margins = o.rvo(act)
        u = A.apply(act, s["collided"], K, rtype, n=k)
        _, _, clear_o = o.step(u, rvo=False)
        col, arr, clear = (t.cpu().numpy() for t in w.step(torch.from_numpy(act).cuda()))
        d = _device(w)
        assert np.array_equal(d["cmd"], A.cmd), (k, np.argwhere(d["cmd"] != A.cmd)[:5])
        ok = np.ones(B * K, bool)
        for b in range(B):
            sl = slice(o.obs_begin[b], o.obs_begin[b + 1])
            if not np.array_equal(d["obs"][sl], o.obs[sl]):
                assert (margins[sl] < 1e-12).any(), (k, b)
                ok[b * K:(b + 1) * K] = False
                excused += 1
        worst = max(worst, float(np.abs(d["states"] - o.states)[ok].max()))
        assert np.array_equal(col[ok], o.collided[ok]) and np.array_equal(arr[ok], o.arrived[ok]), k
        u_ = _ulps(clear, clear_o.astype(np.float32))[ok]
        assert (u_ <= 1).all(), (k, np.flatnonzero(u_ > 1)[:5])
        ulp1 += int((u_ == 1).sum())
    return worst, excused, ulp1


RUNS = {  # robot kinds, K, scenes, motion noise, lidar noise
    "diff_limits": (("diff",), 1, "dyna_obs", False, 0.0),
    "acker_limits": (("acker",), 1, "dyna_obs", False, 0.0),
    "omni_limits": (("omni",), 1, "dyna_obs", False, 0.0),
    "mixed_limits": (("diff", "acker", "omni"), 6, "mixed_swap", False, 0.0),
    "mixed_noise": (("diff", "acker", "omni"), 6, "mixed_swap", True, 0.05),
    "diff_noise": (("diff",), 1, "dyna_obs", True, 0.1),
    "contact_noise": (("diff", "acker", "omni"), 4, "contact", True, 0.05),
}


@pytest.mark.parametrize("run", list(RUNS))
def test_teacher_forced_actuation_matches_the_oracle(run):
    names, K, kind, motion, std = RUNS[run]
    B, steps, seed, lseed = 32, 40, 11, 23
    robots = [_robot(n) for n in names]
    lidar = dict(LIDAR, number=45, scan_offset=(0.1, 0.05, 0.1))
    if kind == "dyna_obs":
        scenes = dyna_obs(B, seed=4)
    elif kind == "mixed_swap":
        scenes = mixed_swap(B, robots=K, seed=4, circles=4)
    else:
        scenes = _contact_scenes(B, K, 31, robots)
    limits = [dict(LIMITS[r.kinematics], alpha=ALPHA if motion else (0.0,) * 4) for r in robots]
    w = WorldBatch(B, robots if len(robots) > 1 else robots[0], lidar, DT)
    w.set_scenes(scenes, seed=13, map_window=1.5)
    w.set_actuation(limits, seed=seed)
    if std:
        w.set_lidar_noise(std, range_min=0.2, seed=lseed)
    o = _oracle(scenes, robots, lidar, seed=13, K=K, window=1.5)
    A = Actuation(pack_actuation(limits, robots), seed, B * K, DT)
    worst, excused, ulp1 = _teacher_forced(w, o, A, scenes, K, steps, lseed, (std, 0.2, lidar["range_max"]), np.random.default_rng(17))
    record(f"world_actuation_teacher_forced_{run}", envs=B, robots=B * K, steps=steps, max_state_err=worst, excused_envs=excused,
           clearance_ulp1=ulp1, collided_at_end=int(o.collided.sum()))
    assert worst <= 1e-12
    w.close()


def test_noise_is_reproducible_from_its_seeds_and_independent_of_B():
    """Two worlds with the same seeds are bitwise equal over 30 steps, another seed differs, a scan repeated without a step is the
    same scan, and a world of the first 16 environments reproduces the first 16 of 48."""
    B, rb = 48, _robot("diff")
    lidar = dict(LIDAR, number=90)
    scenes = dyna_obs(B, seed=8)

    def make(n, mseed, lseed):
        w = WorldBatch(n, rb, lidar, DT)
        w.set_scenes(scenes[:n])
        w.set_actuation([dict(LIMITS["diff"], alpha=ALPHA)], seed=mseed)
        w.set_lidar_noise(0.05, seed=lseed)
        return w

    ws = [make(B, 1, 2), make(B, 1, 2), make(B, 9, 2), make(B, 1, 9), make(16, 1, 2)]
    rng = np.random.default_rng(4)
    differ = [False, False]
    for k in range(30):
        act = torch.from_numpy(_actions(rng, B)).cuda()
        r = [w.scan()[0] for w in ws]
        assert torch.equal(ws[0].scan()[0], r[0])  # a second scan without a step
        assert torch.equal(r[0], r[1]) and torch.equal(r[0][:16], r[4])
        differ[1] |= not torch.equal(r[0], r[3])
        for w in ws:
            w.step(act[:w.B])
        s = [w.states for w in ws]
        assert torch.equal(s[0], s[1]) and torch.equal(s[0][:16], s[4])
        differ[0] |= not torch.equal(s[0], s[2])
    assert all(differ)
    for w in ws:
        w.close()


def test_episode_bank_with_noise_and_limits_is_its_plain_run():
    """S = 24 scenes through 7 slots (max_steps 15) with motion and lidar noise and limits: every slot's scan equals the plain run's
    scan of its scene at the same step, and each scene's results, final state and cmd_prev equal the plain run at its end step, bit
    for bit.  Actions are a function of (scene, step), so both runs feed each scene the same ones."""
    S, slots, T = 24, 7, 15
    rb = _robot("diff")
    lidar = dict(LIDAR, number=60)
    scenes = dyna_obs(S, seed=12)
    for s, sc in enumerate(scenes):  # varied endings: arrival at step 1, collision at step 1, or the timeout
        x, y, _ = sc["start"]
        if s % 3 == 0:
            sc["goal"] = (x, y)
        elif s % 3 == 1:
            sc["obstacles"] = list(sc["obstacles"]) + [dict(center=(x + 1.5, y), radius=0.5)]

    def act_of(s, t):
        a = np.random.default_rng([s, t]).uniform(-2, 2, 2)
        return (a[0] + 1.0, a[1])

    def configure(w):
        w.set_actuation([dict(LIMITS["diff"], alpha=ALPHA)], seed=3)
        w.set_lidar_noise(0.05, seed=4)

    p = WorldBatch(S, rb, lidar, DT)
    p.set_scenes(scenes)
    configure(p)
    plain = []
    for t in range(T):
        r, _, _, h = p.scan(hit=True)
        col, arr, _ = p.step(torch.tensor([act_of(s, t) for s in range(S)], dtype=torch.float32, device="cuda"))
        plain.append(dict(ranges=r.cpu().numpy(), hit=h.cpu().numpy(), col=col.cpu().numpy(), arr=arr.cpu().numpy(),
                          states=p.states.cpu().numpy(), cmd=p.commands().cpu().numpy()))
    end = np.full(S, T)
    for s in range(S):
        for t in range(T):
            if plain[t]["col"][s] or plain[t]["arr"][s]:
                end[s] = t + 1
                break
    e = WorldBatch(S, rb, lidar, DT)
    e.set_episodes(scenes, slots, T)
    configure(e)  # after set_episodes: the settings apply to the bank
    t_slot = np.zeros(slots, np.int64)
    compared = 0
    while int(e.finished().item()) < S:
        scene_of, _ = (x.cpu().numpy() for x in e.slot_scenes())
        r, _, _, h = e.scan(hit=True)
        r, h = r.cpu().numpy(), h.cpu().numpy()
        for b in range(slots):
            s, t = scene_of[b], t_slot[b]
            if t < end[s]:
                assert np.array_equal(r[b], plain[t]["ranges"][s]) and np.array_equal(h[b], plain[t]["hit"][s]), (b, s, t)
                compared += 1
        e.step(torch.tensor([act_of(scene_of[b], min(t_slot[b], T - 1)) for b in range(slots)], dtype=torch.float32, device="cuda"))
        _, reset = (x.cpu().numpy() for x in e.slot_scenes())
        t_slot = np.where(reset != 0, 0, t_slot + 1)
    res = {k: v.cpu().numpy() for k, v in e.episodes().items()}
    states, col, arr = (x.cpu().numpy() for x in e.scene_states())
    cmd = e.commands().cpu().numpy()
    assert np.array_equal(res["end_step"], end)
    for s in range(S):
        pl = plain[end[s] - 1]
        assert res["collided"][s] == pl["col"][s] and res["arrived"][s] == pl["arr"][s], s
        assert np.array_equal(states[s], pl["states"][s]) and np.array_equal(cmd[s], pl["cmd"][s]), s
    record("world_actuation_episode_bank", scenes=S, slots=slots, max_steps=T, scans_compared=compared,
           reasons=np.bincount(res["reason"], minlength=3).tolist())
    assert len(set(end.tolist())) > 1
    p.close()
    e.close()
