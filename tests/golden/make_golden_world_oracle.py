"""Golden runs of the batched world's float64 oracle (oracle/world.py): seeded scenes and seeded actions, free running, every scan
and step output and the state after every step.  tests/test_world_oracle.py replays the same cases and asserts the oracle still
produces these arrays bit for bit.

    python tests/golden/make_golden_world_oracle.py   # writes tests/golden/world_oracle.npz

The oracle is built through ``make_oracle``: the single ``oracle.world.OracleWorld`` where it takes ``fleet``; on a checkout from
before that class existed (commit 02276b2, where the file was recorded), the class that commit's tests used for each kind of case:
``oracle.world`` for circles and convex polygons, and for outlines, reactive obstacles and fleets the oracle module of that kind
under tests/.
"""
import importlib
import inspect
import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from neupan_b200.robot import robot as Robot  # noqa: E402
from neupan_b200.world import dyna_non_obs, dyna_obs, non_obs, pack_behaviors, pack_fleet, pack_scenes_ex  # noqa: E402
from oracle import world as ow  # noqa: E402
from test_gpu_world import _mixed_scenes, _oracle_cfg  # noqa: E402
from test_gpu_world_fleet import _fleet_scenes  # noqa: E402
from test_gpu_world_rvo import ROBOT_KW, _rvo_scenes  # noqa: E402

OUT = os.path.join(HERE, "world_oracle.npz")
B, STEPS = 6, 30
LIDAR = dict(angle_min=-math.pi, angle_max=math.pi, range_min=0.0, range_max=12.0, number=48, scan_offset=(0.1, 0.05, 0.1))


def _still(scenes):
    """The scenes with every obstacle's behaviour removed (constant velocities)."""
    return [dict(sc, obstacles=[{k: v for k, v in ob.items() if k != "behavior"} for ob in sc["obstacles"]]) for sc in scenes]


# name: (oracle of the parent's tests, kinematics, robots per environment, scene builder(robot))
CASES = {
    "circles_diff": ("convex", "diff", 1, lambda rb: dyna_obs(B, seed=1)),
    "convex_acker": ("convex", "acker", 1, lambda rb: _mixed_scenes(B + 2, 9)[2:]),
    "outline_omni": ("outline", "omni", 1, lambda rb: dyna_non_obs(B, seed=2)),
    "outline_diff": ("outline", "diff", 1, lambda rb: non_obs(B, seed=3)),
    "rvo_dyna_obs_diff": ("rvo", "diff", 1, lambda rb: dyna_obs(B, seed=4, behavior="rvo")),
    "rvo_dyna_non_obs_omni": ("rvo", "omni", 1, lambda rb: dyna_non_obs(B, seed=5, behavior="rvo")),
    "rvo_mixed_acker": ("rvo", "acker", 1, lambda rb: _rvo_scenes(B + 1, 23)[1:]),
    "fleet2_diff_rvo": ("fleet", "diff", 2, lambda rb: _fleet_scenes(B, 2, 71, rb)),
    "fleet2_acker": ("fleet", "acker", 2, lambda rb: _still(_fleet_scenes(B, 2, 72, rb))),
    "fleet5_omni_rvo": ("fleet", "omni", 5, lambda rb: _fleet_scenes(B, 5, 73, rb)),
    "fleet5_diff": ("fleet", "diff", 5, lambda rb: _still(_fleet_scenes(B, 5, 74, rb))),
}


def make_oracle(kind, cfg, packed, beh, seed, fleet, K):
    if "fleet" in inspect.signature(ow.OracleWorld).parameters:
        return ow.OracleWorld(cfg, packed, beh, seed, fleet=fleet, K=K)
    if kind == "convex":
        return ow.OracleWorld(cfg, packed[:5])
    cls = importlib.import_module(f"world_{kind}_oracle").OracleWorld  # 02276b2: one module per kind under tests/
    return cls(cfg, packed, fleet, K, beh, seed) if kind == "fleet" else cls(cfg, packed, beh, seed) if kind == "rvo" else cls(cfg, packed)


def _actions(rng, kin, N):
    if kin == "omni":
        return rng.uniform(-1.5, 1.5, (N, 2)).astype(np.float32)
    return np.column_stack([rng.uniform(-1.0, 2.0, N), rng.uniform(-0.5, 0.5, N)]).astype(np.float32)


# per step: the scan, the step and the state after it (for each kind of case, the state its oracle had at 02276b2)
SCAN = ("ranges", "velocity", "hit", "near_tie", "tangent")
STEP = ("collided", "arrived", "clearance")
STATE = {"convex": ("states", "obs"), "outline": ("states", "obs"), "rvo": ("states", "obs", "goal", "draws", "margins"),
         "fleet": ("states", "obs", "goal", "draws", "margins", "robot_clear")}


def run_case(name, oracle=make_oracle):
    """{array name: (STEPS, ...) array} of case ``name``."""
    kind, kin, K, build = CASES[name]
    rb = Robot(10, 0.1, **ROBOT_KW[kin])
    scenes = build(rb)
    packed = pack_scenes_ex(scenes)
    beh = pack_behaviors(scenes) if kind in ("rvo", "fleet") else None
    fleet = pack_fleet(scenes) if kind == "fleet" else None
    o = oracle(kind, _oracle_cfg(rb, LIDAR), packed, beh, 7, fleet, K)
    rng = np.random.default_rng([len(name), K])
    out = {}
    for _ in range(STEPS):
        rec = dict(zip(SCAN, o.scan()))
        rec.update(zip(STEP, o.step(_actions(rng, kin, B * K))))
        rec.update({a: getattr(o, a) for a in STATE[kind]})
        for a, v in rec.items():
            out.setdefault(a, []).append(np.array(v))
    return {a: np.stack(v) for a, v in out.items()}


def main():
    arrays = {}
    for name in CASES:
        for a, v in run_case(name).items():
            arrays[f"{name}/{a}"] = v.astype(np.int16) if a == "hit" else v
        print(name, {a: arrays[f"{name}/{a}"].shape for a in ("ranges",) + STATE[CASES[name][0]]})
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
