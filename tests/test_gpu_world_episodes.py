"""Continuous episodes in the batched world on the GPU.  The central property: every episode is bitwise the plain run of its scene,
truncated at its end.  Each bank runs once in a plain world of S environments with a fresh planner of S environments (every step's
actions, flags, clearances, states, obstacle rows and goals logged), then in episode mode through fewer slots (every step's scene_of
and actions logged); actions, end steps and reasons, per-robot results, final rows and the scene_of trace (against the CPU restatement
tests/world_episode_oracle.py fed the plain flags) must all agree bit for bit.  Also: slots == S, idle slots, set_scenes after
set_episodes, launch counts, repeatability, no host synchronisation, nb_ipath_step_ex and nb_pan_reset_envs_async."""
import math

import numpy as np
import pytest
import torch

from gpu_helpers import make_pan, record
from helpers import CONFIGS, make_inputs, weights_path
from neupan_b200 import InitialPathBatch, MixedPlanner, PlannerBatch, WorldBatch, _lib, run_episodes
from neupan_b200.world import circle_swap, dyna_obs, episode_steps, line_path, maze, mixed_swap, scene_paths
from world_episode_oracle import EpisodeOracle

pytestmark = pytest.mark.gpu

LIDAR = dict(angle_min=-math.pi, angle_max=math.pi, range_min=0.0, range_max=10.0, number=180)
KINDS = ("C4", "C2", "C5")


def _planner(cname, n):
    cfg = CONFIGS[cname]
    return PlannerBatch(n, cfg.T, cfg.dt, 4.0, robot_kwargs=cfg.robot_kwargs, adjust_kwargs=dict(cfg.adjust),
                        pan_kwargs=dict(iter_num=cfg.K, dune_max_num=LIDAR["number"], nrmp_max_num=cfg.M, dune_checkpoint=weights_path(cfg.model),
                                        iter_threshold=0.1, max_points=LIDAR["number"]))


def _robots_of(sc):
    return sc["robots"] if "robots" in sc else [sc]


def _endings(scenes, period=5):
    """Scene s gets ending pattern s mod period: 0 goals at the starts (every robot arrives at step 1), 1 a static circle on every
    start (every robot collides at step 1), 2 goals 2 m ahead (arrivals after a few steps), 3 robot 0 collides at step 1 and the
    others' goals are their starts, 4 as built (the far goal: a timeout, or what the run makes of it)."""
    out = []
    for s, sc in enumerate(scenes):
        sc = dict(sc, obstacles=list(sc["obstacles"]))
        rbs = [dict(r) for r in _robots_of(sc)]
        p = s % period
        for k, r in enumerate(rbs):
            x, y, th = r["start"]
            if p == 0 or (p == 3 and k > 0):
                r["goal"] = (x, y)
            elif p == 2:
                r["goal"] = (x + 2.0 * math.cos(th), y + 2.0 * math.sin(th))
            if p in (1, 3) and (p == 1 or k == 0):
                sc["obstacles"].append(dict(center=(x, y), radius=0.3))
            if p in (0, 2, 3):
                r["path"] = line_path(r["start"], r["goal"])
        if "robots" in sc:
            sc["robots"] = rbs
        else:
            sc.update(rbs[0])
        out.append(sc)
    return out


class _Kit:
    """A world and its planner (a PlannerBatch, or a MixedPlanner of one per kind)."""

    def __init__(self, kinds, n_envs, scenes, K):
        self.kinds, self.K = kinds, K
        self.mixed = len(kinds) > 1
        counts = [sum(1 for sc in scenes[:1] for r in _robots_of(sc) if r.get("type", 0) == t) for t in range(len(kinds))]
        self.pls = [_planner(c, n_envs * counts[t]) for t, c in enumerate(kinds)]
        self.world = WorldBatch(max(n_envs, len(scenes)), [p.robot for p in self.pls] if self.mixed else self.pls[0].robot, LIDAR, self.pls[0].dt)

    def planner(self):
        if not self.mixed:
            return self.pls[0]
        return MixedPlanner([(p, self.world.rows_of_type(t)) for t, p in enumerate(self.pls)])

    def close(self):
        for p in self.pls:
            p.close()
        self.world.close()


def _plain(scenes, kinds, K, steps, seed):
    """The plain run of the bank: per step (actions, collided, arrived, clearance, states, obstacles, goals, draws) as numpy."""
    S = len(scenes)
    kit = _Kit(kinds, S, scenes, K)
    w = kit.world
    w.set_scenes(scenes, seed=seed)
    for t, p in enumerate(kit.pls):
        p.set_initial_paths(scene_paths(scenes, type=t) if kit.mixed else scene_paths(scenes))
    pl = kit.planner()
    beh = any("behavior" in ob for sc in scenes for ob in sc["obstacles"])
    log = {k: [] for k in ("action", "col", "arr", "clear", "states", "obs", "goals", "draws")}
    for _ in range(steps):
        r, v, sc = w.scan()
        a, _ = pl.forward(w.states, r, sc, scan_offset=w.scan_offset, scan_velocity=v)
        col, arr, clear = w.step(a)
        g, d = w.goals() if beh else (torch.zeros(1), torch.zeros(1))
        for k, x in zip(log, (a, col, arr, clear, w.states, w.obstacles(), g, d)):
            log[k].append(x.cpu().numpy())
    kit.close()
    return {k: np.stack(v) for k, v in log.items()}, w.O


def _episodes(scenes, kinds, K, slots, max_steps, seed):
    """The episode run: per step scene_of (before the step) and actions; then the results and the bank's rows."""
    S = len(scenes)
    kit = _Kit(kinds, slots, scenes, K)
    w = kit.world
    w.set_episodes(scenes, slots, max_steps, seed=seed)
    pl = kit.planner()
    if kit.mixed:
        pl.load_bank(scenes)
    else:
        pl.load_bank(scene_paths(scenes))
    trace, resets, actions = [], [], []
    while int(w.finished().item()) < S:
        scene_of, reset = w.slot_scenes()
        r, v, sc = w.scan()
        a, _ = pl.forward(w.states, r, sc, scan_offset=w.scan_offset, scan_velocity=v, scene_of=scene_of, reset=reset)
        w.step(a)
        trace.append(scene_of.cpu().numpy()); resets.append(reset.cpu().numpy()); actions.append(a.cpu().numpy())
        assert len(trace) <= S * max_steps
    res = {k: v.cpu().numpy() for k, v in w.episodes().items()}
    states, col, arr = (x.cpu().numpy() for x in w.scene_states())
    beh = any("behavior" in ob for sc in scenes for ob in sc["obstacles"])
    g, d = w.goals() if beh else (torch.zeros(1), torch.zeros(1))
    final = dict(states=states, col=col, arr=arr, obs=w.obstacles().cpu().numpy(), goals=g.cpu().numpy(), draws=d.cpu().numpy())
    kit.close()
    return np.asarray(trace), np.asarray(resets), np.asarray(actions), res, final


def _check_bank(name, scenes, kinds, K, slots, max_steps, seed=7):
    S = len(scenes)
    plain, O = _plain(scenes, kinds, K, max_steps, seed)
    trace, resets, actions, res, final = _episodes(scenes, kinds, K, slots, max_steps, seed)
    # the CPU restatement fed the plain flags: the same scene_of trace and results
    rows = lambda s: slice(s * K, (s + 1) * K)
    flags = lambda s, t: (plain["col"][t - 1][rows(s)], plain["arr"][t - 1][rows(s)], plain["clear"][t - 1][rows(s)])
    oracle = EpisodeOracle(S, slots, K, max_steps)
    want_trace = oracle.run(flags)
    assert np.array_equal(trace, want_trace)
    assert np.array_equal(res["end_step"], oracle.end_step) and np.array_equal(res["reason"], oracle.reason)
    assert np.array_equal(res["slot"], oracle.slot)
    assert np.array_equal(res["steps_to_arrive"], oracle.arrive_step)
    assert np.array_equal(res["min_clearance"].view(np.int32), oracle.min_clearance.view(np.int32))
    assert np.array_equal(res["collided"], oracle.collided.astype(bool)) and np.array_equal(res["arrived"], oracle.arrived.astype(bool))
    # every action of scene s at its step t is the plain run's action of environment s at step t
    start = {}
    compared = 0
    for k in range(len(trace)):
        for b in range(slots):
            s = int(trace[k][b])
            if resets[k][b]:
                start[s] = k
            t = k - start[s] + 1
            if t <= res["end_step"][s]:
                assert np.array_equal(actions[k][b * K:(b + 1) * K].view(np.int32), plain["action"][t - 1][rows(s)].view(np.int32)), (name, s, t)
                compared += 1
    # each scene's final rows: the plain run's after its end step
    for s in range(S):
        t = int(res["end_step"][s])
        assert np.array_equal(final["states"][rows(s)], plain["states"][t - 1][rows(s)])
        assert np.array_equal(final["col"][rows(s)], plain["col"][t - 1][rows(s)]) and np.array_equal(final["arr"][rows(s)], plain["arr"][t - 1][rows(s)])
    obs_begin = np.cumsum([0] + [len(sc["obstacles"]) for sc in scenes])
    for s in range(S):
        t, o = int(res["end_step"][s]), slice(obs_begin[s], obs_begin[s + 1])
        assert np.array_equal(final["obs"][o], plain["obs"][t - 1][o])
        if final["goals"].ndim == 2:
            assert np.array_equal(final["goals"][o], plain["goals"][t - 1][o]) and np.array_equal(final["draws"][o], plain["draws"][t - 1][o])
    per_slot = [len({int(s) for s in trace[:, b]}) for b in range(slots)]
    counts = dict(arrived=int(((res["reason"] == 1) & np.array([res["arrived"][rows(s)].all() for s in range(S)])).sum()),
                  collision=int(np.array([res["collided"][rows(s)].any() for s in range(S)]).sum()), timeout=int((res["reason"] == 2).sum()))
    record(f"episodes_{name}", S=S, slots=slots, K=K, max_steps=max_steps, steps=len(trace), actions_compared=compared,
           scenes_per_slot=per_slot, **counts)
    assert min(per_slot) >= 3, per_slot  # every slot reused at least twice
    assert counts["arrived"] > 0 and counts["collision"] > 0 and counts["timeout"] > 0, counts


def test_dyna_obs_rvo_diff():
    _check_bank("dyna_obs_rvo", _endings(dyna_obs(20, seed=11, behavior="rvo")), ("C4",), 1, 4, 14)


def test_circle_swap_k4_acker():
    _check_bank("circle_swap_k4", _endings(circle_swap(15, robots=4, radius=6.0, seed=5)), ("C2",), 4, 3, 12)


def test_mixed_swap_k3():
    _check_bank("mixed_swap_k3", _endings(mixed_swap(15, robots=3, radius=6.0, seed=5)), KINDS, 3, 3, 12)


def test_maze_map():
    _check_bank("maze", _endings(maze(15, cells=(3, 3), seed=3, layouts=3)), ("C4",), 1, 3, 12)


# ---- edge cases ------------------------------------------------------------------------------------------------------------

def _dyna(S=8):
    return _endings(dyna_obs(S, seed=4, behavior="rvo"))


def test_slots_equal_to_scenes_is_the_plain_run_truncated():
    scenes = _dyna(5)
    plain, _ = _plain(scenes, ("C4",), 1, 10, 7)
    trace, resets, actions, res, final = _episodes(scenes, ("C4",), 1, 5, 10, 7)
    assert (trace == np.arange(5)).all() and resets[0].all() and not resets[1:].any()
    for s in range(5):
        t = int(res["end_step"][s])
        assert np.array_equal(actions[:t, s], plain["action"][:t, s])
        assert np.array_equal(final["states"][s], plain["states"][t - 1][s])
    assert res["end_step"][0] == 1 and res["reason"][0] == 1 and res["steps_to_arrive"][0] == 1  # a scene that arrives at step 1


def _episode_world(scenes, slots, max_steps, seed=7):
    pl = _planner("C4", slots)
    w = WorldBatch(len(scenes), pl.robot, LIDAR, pl.dt)
    w.set_episodes(scenes, slots, max_steps, seed=seed)
    pl.load_bank(scene_paths(scenes))
    return w, pl


def test_idle_slots_leave_their_scene_untouched_and_runs_repeat():
    scenes = _dyna(6)
    outs = []
    for _ in range(2):
        w, pl = _episode_world(scenes, 4, 10)
        trace = []
        for _ in range(30):
            sc, _ = w.slot_scenes()
            trace.append(sc.cpu().numpy())
            episode_steps(pl, w, 1)
        before = [x.cpu().numpy() for x in w.scene_states()] + [w.obstacles().cpu().numpy(), w.goals()[0].cpu().numpy()]
        res = {k: v.cpu().numpy() for k, v in w.episodes().items()}
        assert int(w.finished().item()) == 6
        episode_steps(pl, w, 5)  # every slot idle now
        after = [x.cpu().numpy() for x in w.scene_states()] + [w.obstacles().cpu().numpy(), w.goals()[0].cpu().numpy()]
        for x, y in zip(before, after):
            assert np.array_equal(x, y)
        res2 = {k: v.cpu().numpy() for k, v in w.episodes().items()}
        assert all(np.array_equal(res[k], res2[k]) for k in res)
        outs.append((np.asarray(trace), res, before))
        pl.close(); w.close()
    assert np.array_equal(outs[0][0], outs[1][0])
    assert all(np.array_equal(outs[0][1][k], outs[1][1][k]) for k in outs[0][1])
    assert all(np.array_equal(x, y) for x, y in zip(outs[0][2], outs[1][2]))


def test_run_episodes_and_no_host_synchronisation():
    scenes = _dyna(6)
    w, pl = _episode_world(scenes, 3, 8)
    out = run_episodes(pl, w, check_every=4)
    assert out["steps"] % 4 == 0 and (out["end_step"].cpu().numpy() >= 1).all() and (out["reason"].cpu().numpy() > 0).all()
    w.set_episodes(scenes, 3, 8, seed=7)
    pl.load_bank(scene_paths(scenes))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        episode_steps(pl, w, 4)
        episode_steps(pl, w, 2, blind=True)
        episode_steps(pl, w, 2, velocities=False)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    pl.close(); w.close()


def test_set_scenes_after_set_episodes_is_a_fresh_world_and_launch_counts():
    scenes = _dyna(4)
    pl = _planner("C4", 4)
    fresh = WorldBatch(4, pl.robot, LIDAR, pl.dt)
    used = WorldBatch(4, pl.robot, LIDAR, pl.dt)
    used.set_episodes(scenes, 2, 5, seed=7)
    act = torch.full((2, 2), 0.3, device="cuda")
    for _ in range(6):
        used.scan(); used.step(act)
    lib = _lib.load()
    n0 = lib.nb_launch_count()
    used.states
    used.step(act)
    torch.cuda.synchronize()
    assert lib.nb_launch_count() - n0 == 1 + 3  # the slot gather; rvo, step and the advance kernel
    fresh.set_scenes(scenes, seed=7)
    used.set_scenes(scenes, seed=7)
    assert used.N == 4 and used.S is None
    a = torch.full((4, 2), 0.4, device="cuda")
    for _ in range(5):
        outs = []
        for w in (fresh, used):
            n0 = lib.nb_launch_count()
            r, v, _, h = w.scan(hit=True)
            c, ar, cl = w.step(a)
            outs.append([x.cpu().numpy() for x in (r, v, h, c, ar, cl, w.states, w.obstacles())])
            assert lib.nb_launch_count() - n0 == 3  # scan, rvo, step
        assert all(np.array_equal(x, y) for x, y in zip(*outs))
    pl.close(); fresh.close(); used.close()


# ---- nb_ipath_step_ex and nb_pan_reset_envs_async ----------------------------------------------------------------------

def test_ipath_step_ex_identity_and_permutation():
    scenes = dyna_obs(6, seed=9)
    paths = scene_paths(scenes)
    rng = np.random.default_rng(0)
    mk = lambda: InitialPathBatch(10, 0.1, "diff", max_envs=6)
    plain, ident, perm = mk(), mk(), mk()
    for p in (plain, ident, perm):
        p.set_initial_paths(paths)
    order = torch.tensor([3, 0, 5, 1, 4, 2], dtype=torch.int32, device="cuda")
    for step in range(8):
        st = torch.tensor([[sc["start"][0] + 0.3 * step, sc["start"][1], sc["start"][2]] for sc in scenes], dtype=torch.float64, device="cuda")
        cv = torch.from_numpy(rng.uniform(-1, 1, (6, 2, 10)).astype(np.float32)).cuda()
        a = plain.step(st, cv, 4.0)
        b = ident.step(st, cv, 4.0, env_index=torch.arange(6, dtype=torch.int32, device="cuda"))
        c = perm.step(st[order.long()], cv[order.long()], 4.0, env_index=order)
        for x, y, z in zip(a, b, c):
            assert torch.equal(x, y) and torch.equal(x[order.long()], z)
    sa, sc_ = plain.read_state(), perm.read_state()
    assert all(torch.equal(sa[k], sc_[k]) for k in ("curve_index", "point_index", "arrive_flag")) and np.array_equal(sa["points"], sc_["points"])
    for p in (plain, ident, perm):
        p.close()


def test_pan_reset_envs():
    cfg = CONFIGS["C4"]
    B = 6
    inp = make_inputs(cfg, B=B, N=60, scene="obstacles")
    t = {k: (None if v is None else torch.from_numpy(np.ascontiguousarray(v)).cuda()) for k, v in inp.items()}
    args = (t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"])

    def run(reset):
        pan = make_pan(cfg, N=60, max_envs=B, iter_threshold=0.1)
        outs = []
        with torch.no_grad():
            for k in range(4):
                if k == 2:
                    reset(pan)
                S, U, D = pan(*args)
                outs.append([x.cpu().numpy() for x in (S, U, D)])
        pan.close()
        return outs

    def masked(m):
        return lambda pan: pan.reset_envs(torch.tensor(m, dtype=torch.int32, device="cuda"))

    full = run(lambda pan: pan.reset_state())
    ones = run(masked([1] * B))
    none = run(lambda pan: None)
    half = run(masked([1, 0, 1, 0, 0, 1]))
    for a, b in zip(full, ones):
        assert all(np.array_equal(x, y) for x, y in zip(a, b))
    m = np.array([1, 0, 1, 0, 0, 1], bool)
    for f, n, h in zip(full, none, half):
        for x, y, z in zip(f, n, h):
            assert np.array_equal(z[m], x[m]) and np.array_equal(z[~m], y[~m])
