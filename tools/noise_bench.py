"""Actuation limits and noise in the batched world (nb_world_set_actuation, nb_world_set_lidar_noise), on the device; prints JSON lines.

    python tools/noise_bench.py [--envs 128] [--steps 200] [--beams 1080] [--kernel-envs 4096] [--kernel-steps 50] [--rounds 3]

Closed loop: seeded dyna_obs(--envs) scenes (20 constant-velocity circles, neupan_b200.world.dyna_obs) driven by C4's PlannerBatch
(its robot, adjust values and K, the scans decimated to C4's N = 500 points) through rollout for --steps steps, once per
range_std in {0, 0.02, 0.05, 0.1} m and alpha in {0, 0.03} (all four alpha equal).  Every run sets the actuation limits to the
planner robot's own speed and acceleration bounds (so the planner's commands already respect them) with motion seed 1 and lidar seed
2; it reports collisions, arrivals and the median of the robots' minimum clearance.  Kernels: dyna_obs(--kernel-envs) at --beams
beams, scan and step (zero action) timed separately with CUDA events over --kernel-steps calls, for a world without the calls
("off") and one with limits, alpha 0.03 and range_std 0.05 ("on"), alternated --rounds times; the medians and the spread over the
rounds.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=128)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--beams", type=int, default=1080)
    ap.add_argument("--kernel-envs", type=int, default=4096)
    ap.add_argument("--kernel-steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import numpy as np
    import torch

    from helpers import CONFIGS, weights_path
    from neupan_b200 import PlannerBatch, WorldBatch, rollout
    from neupan_b200.world import dyna_obs, scene_paths
    from world_bench import _card

    if not torch.cuda.is_available():
        raise SystemExit("noise_bench.py needs a CUDA device")
    card = _card()
    cfg = CONFIGS["C4"]
    lidar = dict(angle_min=-math.pi, angle_max=math.pi, range_min=0.0, range_max=10.0, number=args.beams)
    B = args.envs
    scenes = dyna_obs(B, seed=2024)
    pl = PlannerBatch(B, cfg.T, cfg.dt, 4.0, robot_kwargs=cfg.robot_kwargs, adjust_kwargs=dict(cfg.adjust),
                      pan_kwargs=dict(iter_num=cfg.K, dune_max_num=cfg.N, nrmp_max_num=cfg.M, dune_checkpoint=weights_path(cfg.model),
                                      iter_threshold=0.1, max_points=cfg.N))
    rb = pl.robot
    vmax, amax = rb.max_speed.reshape(-1).tolist(), rb.max_acce.reshape(-1).tolist()
    limits = dict(vel_min=(-vmax[0], -vmax[1]), vel_max=tuple(vmax), acce=tuple(amax))
    world = WorldBatch(B, rb, lidar, pl.dt)
    for alpha in (0.0, 0.03):
        for std in (0.0, 0.02, 0.05, 0.1):
            world.set_scenes(scenes)
            world.set_actuation([dict(limits, alpha=(alpha,) * 4)], seed=1)
            world.set_lidar_noise(std, seed=2)
            pl.set_initial_paths(scene_paths(scenes))
            pl.reset()
            out = rollout(pl, world, args.steps)
            mc = out["min_clearance"].cpu().numpy()
            print(json.dumps(dict(metric="closed loop under actuation noise", scene="dyna_obs", envs=B, steps=args.steps, beams=args.beams,
                                  range_std=std, alpha=alpha, vel_max=vmax, acce=amax, collisions=int(out["collided"].sum()),
                                  arrivals=int(out["arrived"].sum()), median_min_clearance=float(np.median(mc)), **card)), flush=True)
    world.close()
    pl.close()

    Bk = args.kernel_envs
    kscenes = dyna_obs(Bk, seed=2024)
    worlds = {"off": WorldBatch(Bk, rb, lidar, cfg.dt), "on": WorldBatch(Bk, rb, lidar, cfg.dt)}
    for w in worlds.values():
        w.set_scenes(kscenes)
    worlds["on"].set_actuation([dict(limits, alpha=(0.03,) * 4)], seed=1)
    worlds["on"].set_lidar_noise(0.05, seed=2)
    zero = torch.zeros(Bk, 2, device="cuda")

    def timed(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.kernel_steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.kernel_steps

    ms = {k: dict(scan=[], step=[]) for k in worlds}
    for _ in range(args.rounds):
        for name, w in worlds.items():
            ms[name]["scan"].append(timed(w.scan))
            ms[name]["step"].append(timed(lambda: w.step(zero)))
    summary = {f"ms_{part}_{name}": float(np.median(v)) for name, d in ms.items() for part, v in d.items()}
    spread = {f"ms_{part}_{name}_range": [min(v), max(v)] for name, d in ms.items() for part, v in d.items()}
    print(json.dumps(dict(metric="world scan / step kernels with actuation and noise off and on", scene="dyna_obs", envs=Bk, beams=args.beams,
                          calls=args.kernel_steps, rounds=args.rounds, **summary, **spread, **card)), flush=True)
    for w in worlds.values():
        w.close()


if __name__ == "__main__":
    main()
