"""Every scan, step, contact and RVO kernel instantiation of the batched world on the GPU, through the configurations of MATRIX
(tests/test_world_variants.py, which checks that they reach all of them): teacher-forced parity of each plain configuration with the
composed float64 oracles (ContactOracleWorld over the map-motion, map and mixed oracles, with Actuation and lidar_noise from
tests/world_actuation_oracle.py); each episode configuration as a bank that equals the plain run of its scenes bit for bit; and
actuation at its neutral settings bitwise equal to the kernel it stands in for.  Every scan and step launches the kernels the
dispatch mirror names (nb_launch_count)."""
import numpy as np
import pytest
import torch

from gpu_helpers import record
from neupan_b200 import WorldBatch, _lib
from neupan_b200.world import pack_actuation, pack_robot_types, pack_scenes_ex
from test_gpu_world import LIDAR, _ulps
from test_gpu_world_actuation import ALPHA, LIMITS
from test_gpu_world_contact import _oracle
from test_gpu_world_mixed import _mixed_actions
from test_world_variants import B_BANK, B_PLAIN, MATRIX, dispatch, flags_of, variant_scenes
from world_actuation_oracle import Actuation, lidar_noise

pytestmark = pytest.mark.gpu

DT = 0.1
WINDOW = 1.5
LIDAR45 = dict(LIDAR, number=45, scan_offset=(0.1, 0.05, 0.1))
RANGE_STD, RANGE_MIN = 0.05, 0.2
SEED_SCENES, SEED_MOTION, SEED_LIDAR = 13, 11, 23


def _limits(robots):
    return [dict(LIMITS[r.kinematics], alpha=ALPHA) for r in robots]


def _world(name, scenes, robots, slots=None, max_steps=None, neutral=False, settings=True):
    """A world of ``scenes`` (a bank through ``slots`` slots if given, else a plain world) with MATRIX[name]'s actuation and lidar
    noise; ``neutral``: every actuation key at its default and range_std 0 instead; ``settings`` False: neither call."""
    cfg = MATRIX[name]
    w = WorldBatch(len(scenes), robots if len(robots) > 1 else robots[0], LIDAR45, DT)
    if slots:
        w.set_episodes(scenes, slots, max_steps, seed=SEED_SCENES, map_window=WINDOW)
    else:
        w.set_scenes(scenes, seed=SEED_SCENES, map_window=WINDOW)
    if neutral:
        w.set_actuation([{} for _ in robots], seed=SEED_MOTION)
        w.set_lidar_noise(0.0, seed=SEED_LIDAR)
    elif settings:
        if cfg["act"]:
            w.set_actuation(_limits(robots), seed=SEED_MOTION)
        if cfg["noise"]:
            w.set_lidar_noise(RANGE_STD, range_min=RANGE_MIN, seed=SEED_LIDAR)
    return w


def _counted(call):
    """call()'s result and the kernels it launched."""
    lib = _lib.load()
    n0 = lib.nb_launch_count()
    out = call()
    return out, lib.nb_launch_count() - n0


def _device(w, goals):
    c, a = w.flags()
    d = dict(obs=w.obstacles().cpu().numpy(), states=w.states.cpu().numpy(), collided=c.cpu().numpy(), arrived=a.cpu().numpy(),
             cmd=w.commands().cpu().numpy())
    if goals:
        d["goal"], d["draws"] = (x.cpu().numpy() for x in w.goals())
    return d


# ---- 2. teacher-forced parity of every plain configuration ---------------------------------------------------------------------

@pytest.mark.parametrize("name", [n for n, c in MATRIX.items() if not c["ep"]])
def test_teacher_forced_variant_matches_the_oracle(name):
    """30 steps of B = 32 environments of a mixed fleet (K = 3: diff, acker, omni): before every step the oracle takes the device's
    obstacles, goals, states, flags and cmd_prev.  Hits exact, ranges within 1 ulp (after lidar_noise), velocities within rtol 1e-6,
    cmd_prev bitwise, flags exact, states within 1e-12, clearances within 1 ulp; obstacle rows and goals bitwise, except in an
    environment where a reactive obstacle's decision margin is below 1e-12 (the reactive tests' excuse, which excuses its robots)."""
    cfg = MATRIX[name]
    B, steps = B_PLAIN, 30
    scenes, robots, K = variant_scenes(name, B)
    flags = flags_of(name, scenes)
    step_k, scan_k = dispatch(**flags)
    rtype = pack_robot_types(scenes)
    kins = [r.kinematics for r in robots]
    w = _world(name, scenes, robots)
    o = _oracle(scenes, robots, LIDAR45, seed=SEED_SCENES, K=K, window=WINDOW)
    A = Actuation(pack_actuation(_limits(robots), robots), SEED_MOTION, B * K, DT) if cfg["act"] else None
    rng = np.random.default_rng(17)
    worst, excused, ulp1 = 0.0, 0, 0
    for k in range(steps):
        s = _device(w, flags["rvo"])
        o.obs[:], o.states[:], o.collided[:], o.arrived[:] = s["obs"], s["states"], s["collided"], s["arrived"]
        if flags["rvo"]:
            o.goal[:], o.draws[:] = s["goal"], s["draws"]
        if A is not None:
            A.cmd[:] = s["cmd"]
        out, launched = _counted(lambda: w.scan(hit=True))
        assert launched == len(scan_k), (k, launched, scan_k)
        ranges, vel, hit = (t.cpu().numpy() for t in (out[0], out[1], out[3]))
        r64, v64, h64, _, _ = o.scan()
        assert np.array_equal(hit, h64), (k, np.argwhere(hit != h64)[:5])
        if cfg["noise"]:
            r64 = lidar_noise(r64, h64, K, SEED_LIDAR, RANGE_STD, RANGE_MIN, LIDAR45["range_max"], n=k)
        assert (_ulps(ranges, r64.astype(np.float32)) <= 1).all(), k
        assert np.allclose(vel, v64, rtol=1e-6, atol=0), k
        act = _mixed_actions(rng, kins, rtype, s["states"], K)
        margins = o.rvo(act)
        u = A.apply(act, s["collided"], K, rtype, n=k) if A is not None else act
        _, _, clear_o = o.step(u, rvo=False)
        out, launched = _counted(lambda: w.step(torch.from_numpy(act).cuda()))
        assert launched == len(step_k), (k, launched, step_k)
        col, arr, clear = (t.cpu().numpy() for t in out)
        d = _device(w, flags["rvo"])
        if A is not None:
            assert np.array_equal(d["cmd"], A.cmd), (k, np.argwhere(d["cmd"] != A.cmd)[:5])
        else:
            assert not d["cmd"].any()
        ok = np.ones(B * K, bool)
        for b in range(B):
            sl = slice(o.obs_begin[b], o.obs_begin[b + 1])
            same = np.array_equal(d["obs"][sl], o.obs[sl])
            if flags["rvo"]:
                same = same and np.array_equal(d["goal"][sl], o.goal[sl]) and np.array_equal(d["draws"][sl], o.draws[sl])
            if not same:
                assert (margins[sl] < 1e-12).any(), (k, b)
                ok[b * K:(b + 1) * K] = False
                excused += 1
        worst = max(worst, float(np.abs(d["states"] - o.states)[ok].max()))
        assert np.array_equal(col[ok], o.collided[ok]) and np.array_equal(arr[ok], o.arrived[ok]), k
        u_ = _ulps(clear, clear_o.astype(np.float32))[ok]
        assert (u_ <= 1).all(), (k, np.flatnonzero(u_ > 1)[:5])
        ulp1 += int((u_ == 1).sum())
    record(f"world_variants_teacher_forced_{name}", envs=B, robots=B * K, steps=steps, kernels=step_k + scan_k, max_state_err=worst,
           excused_envs=excused, clearance_ulp1=ulp1, collided_at_end=int(o.collided.sum()), arrived_at_end=int(o.arrived.sum()))
    assert worst <= 1e-12
    w.close()


# ---- 3. every episode configuration is its plain run ---------------------------------------------------------------------------

def _act_of(s, t, K):
    """The actions of scene s at step t of its episode: a function of (scene, step) alone."""
    a = np.random.default_rng([s, t]).uniform(-1.0, 1.0, (K, 2))
    return np.column_stack([2.0 * a[:, 0] + 1.0, a[:, 1]]).astype(np.float32)


@pytest.mark.parametrize("name", [n for n, c in MATRIX.items() if c["ep"]])
def test_episode_bank_is_its_plain_run(name):
    """S = 24 scenes of K = 2 robots through 7 slots (max_steps 20) and the plain run of the same scenes with the same settings:
    every live slot's scan (ranges, velocities, hits) equals the plain scan of its scene at that step, and each scene's end step,
    reason, flags, final states, cmd_prev, obstacle rows (and goals and draws of reactive obstacles) equal the plain run at its end
    step, bit for bit.  A third of the scenes end by arrival at step 1; the others end by collision or the timeout."""
    S, slots, T = B_BANK, 7, 20
    scenes, robots, K = variant_scenes(name, S)
    flags = flags_of(name, scenes)
    step_k, scan_k = dispatch(**flags)
    plain_step_k, plain_scan_k = dispatch(**dict(flags, ep=False))
    rvo = flags["rvo"]
    p = _world(name, scenes, robots)
    scans, hist = [], [_device(p, rvo)]
    for t in range(T):
        (r, v, _, h), n_scan = _counted(lambda: p.scan(hit=True))
        scans.append(dict(ranges=r.cpu().numpy(), vel=v.cpu().numpy(), hit=h.cpu().numpy()))
        act = np.concatenate([_act_of(s, t, K) for s in range(S)])
        _, n_step = _counted(lambda: p.step(torch.from_numpy(act).cuda()))
        assert (n_scan, n_step) == (len(plain_scan_k), len(plain_step_k)), t
        hist.append(_device(p, rvo))
    end = np.full(S, T)
    for s in range(S):
        rows = slice(s * K, (s + 1) * K)
        for t in range(1, T + 1):
            if ((hist[t]["collided"][rows] != 0) | (hist[t]["arrived"][rows] != 0)).all():
                end[s] = t
                break
    e = _world(name, scenes, robots, slots, T)
    t_slot = np.zeros(slots, np.int64)
    compared = 0
    for _ in range(S * T):
        if int(e.finished().item()) >= S:
            break
        scene_of, _ = (x.cpu().numpy() for x in e.slot_scenes())
        (r, v, _, h), n_scan = _counted(lambda: e.scan(hit=True))
        assert n_scan == len(scan_k)
        r, v, h = r.cpu().numpy(), v.cpu().numpy(), h.cpu().numpy()
        for b in range(slots):
            s, t = scene_of[b], t_slot[b]
            if t < end[s]:
                q, n = slice(b * K, (b + 1) * K), slice(s * K, (s + 1) * K)
                pl = scans[t]
                assert np.array_equal(r[q], pl["ranges"][n]) and np.array_equal(h[q], pl["hit"][n]) and np.array_equal(v[q], pl["vel"][n]), (b, s, t)
                compared += 1
        act = np.concatenate([_act_of(int(scene_of[b]), int(min(t_slot[b], T - 1)), K) for b in range(slots)])
        _, n_step = _counted(lambda: e.step(torch.from_numpy(act).cuda()))
        assert n_step == len(step_k)
        _, reset = (x.cpu().numpy() for x in e.slot_scenes())
        t_slot = np.where(reset != 0, 0, t_slot + 1)
    assert int(e.finished().item()) == S
    res = {k: v.cpu().numpy() for k, v in e.episodes().items()}
    states, col, arr = (x.cpu().numpy() for x in e.scene_states())
    cmd, obs = e.commands().cpu().numpy(), e.obstacles().cpu().numpy()
    goal, draws = (x.cpu().numpy() for x in e.goals()) if rvo else (None, None)
    assert np.array_equal(res["end_step"], end)
    ob = pack_scenes_ex(scenes)[0]
    ends = dict(arrived=0, collided=0, timeout=0)
    for s in range(S):
        h = hist[end[s]]
        rows, sl = slice(s * K, (s + 1) * K), slice(ob[s], ob[s + 1])
        done = ((h["collided"][rows] != 0) | (h["arrived"][rows] != 0)).all()
        assert res["reason"][s] == (1 if done else 2), s
        assert np.array_equal(res["collided"][rows], h["collided"][rows] != 0) and np.array_equal(res["arrived"][rows], h["arrived"][rows] != 0), s
        assert np.array_equal(col[rows], h["collided"][rows]) and np.array_equal(arr[rows], h["arrived"][rows]), s
        assert np.array_equal(states[rows], h["states"][rows]) and np.array_equal(cmd[rows], h["cmd"][rows]), s
        assert np.array_equal(obs[sl], h["obs"][sl]), s
        if rvo:
            assert np.array_equal(goal[sl], h["goal"][sl]) and np.array_equal(draws[sl], h["draws"][sl]), s
        ends["timeout" if not done else "arrived" if (h["arrived"][rows] != 0).all() else "collided"] += 1
    record(f"world_variants_episode_bank_{name}", scenes=S, slots=slots, max_steps=T, kernels=step_k + scan_k, scans_compared=compared,
           **ends)
    assert ends["arrived"] > 0 and ends["collided"] + ends["timeout"] > 0 and len(set(end.tolist())) > 1
    p.close()
    e.close()


# ---- 4. neutral actuation is bitwise the kernel it stands in for ---------------------------------------------------------------

def _outputs(w, act, ep):
    out = [t for t in w.scan(hit=True) if torch.is_tensor(t)] + list(w.step(act))
    out += [w.states, w.obstacles()] + list(w.flags())
    return out + (list(w.slot_scenes()) + [w.finished()] if ep else [])


@pytest.mark.parametrize("name", [n for n, c in MATRIX.items() if c["act"]])
def test_neutral_actuation_is_bitwise_the_kernel_it_stands_in_for(name):
    """The configuration's scenes with every actuation key at its default and range_std 0 (its actuation kernel) next to a world
    without either call (the step kernel that kernel stands in for): scans, steps, states, obstacles and flags (and the slots' scenes
    in episode mode) are bitwise equal over 30 steps, with the same number of launches; cmd_prev is the action, 0 once collided."""
    cfg = MATRIX[name]
    B = B_BANK if cfg["ep"] else B_PLAIN
    scenes, robots, K = variant_scenes(name, B)
    flags = flags_of(name, scenes)
    act_k, plain_k = dispatch(**dict(flags, noise=False))[0], dispatch(**dict(flags, act=False, noise=False))[0]
    assert act_k != plain_k
    kw = dict(slots=7, max_steps=20) if cfg["ep"] else {}
    plain, neutral = _world(name, scenes, robots, settings=False, **kw), _world(name, scenes, robots, neutral=True, **kw)
    rng = np.random.default_rng(2)
    for k in range(30):
        act = torch.from_numpy(np.column_stack([rng.uniform(-1.0, 2.5, plain.N), rng.uniform(-0.5, 0.5, plain.N)]).astype(np.float32)).cuda()
        frozen = None if cfg["ep"] else plain.flags()[0].bool()[:, None]
        a, n_plain = _counted(lambda: _outputs(plain, act, cfg["ep"]))
        b, n_neutral = _counted(lambda: _outputs(neutral, act, cfg["ep"]))
        assert n_plain == n_neutral, k
        for i, (x, y) in enumerate(zip(a, b)):
            assert torch.equal(x, y), (k, i)
        if frozen is not None:
            assert torch.equal(neutral.commands(), torch.where(frozen, 0.0, act.double())), k
    record(f"world_variants_neutral_{name}", envs=B, steps=30, actuation_kernel=act_k, stands_in_for=plain_k)
    plain.close()
    neutral.close()
