"""Continuous episodes against fixed-length rollout batches on the same bank of scenes, and prints one JSON line.

    python tools/episode_bench.py [--scenes 16384] [--slots 4096] [--max-steps 150] [--beams 1080] [--check-every 16]
                                  [--profile-steps 20]

Bank: seeded dyna_obs(behavior="rvo") scenes (neupan_b200.world.dyna_obs: 20 reactive circles, the robot crossing the box).  Planner:
PlannerBatch with C4's robot, adjust values and K, scans decimated to C4's N = 500 points, iter_threshold 0.1 (the yaml default).
Legs, each timed with CUDA events around the whole leg (host included):
  rollout   ceil(S / B) batches of B environments, each set_scenes + set_initial_paths + rollout(max_steps) -- the host-driven way
  episodes  set_episodes(bank, B slots, max_steps) + load_bank + run_episodes(check_every)
Planner steps (rows x steps) spent on finished episodes: for the rollout batches, every row's steps after its scene's episode ended
(the end steps of the episode run, which equal the plain run's bit for bit) plus the empty rows of a short last batch; for the
episode run, the steps of idle slots.  Then a separate run of --profile-steps episode steps under torch.profiler gives the device
time of world_advance_kernel per step.  The card's name and power limit are read in the same run.
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
    ap.add_argument("--scenes", type=int, default=16384)
    ap.add_argument("--slots", type=int, default=4096)
    ap.add_argument("--max-steps", type=int, default=150)
    ap.add_argument("--beams", type=int, default=1080)
    ap.add_argument("--check-every", type=int, default=16)
    ap.add_argument("--profile-steps", type=int, default=20)
    args = ap.parse_args()

    import torch

    from helpers import CONFIGS, weights_path
    from neupan_b200 import PlannerBatch, WorldBatch, rollout, run_episodes
    from neupan_b200.world import dyna_obs, episode_steps, scene_paths
    from world_bench import _card

    if not torch.cuda.is_available():
        raise SystemExit("episode_bench.py needs a CUDA device")
    S, B, T = args.scenes, args.slots, args.max_steps
    cfg = CONFIGS["C4"]
    lidar = dict(angle_min=-math.pi, angle_max=math.pi, range_min=0.0, range_max=10.0, number=args.beams)
    scenes = dyna_obs(S, seed=2024, behavior="rvo")
    pl = PlannerBatch(B, cfg.T, cfg.dt, 4.0, robot_kwargs=cfg.robot_kwargs, adjust_kwargs=dict(cfg.adjust),
                      pan_kwargs=dict(iter_num=cfg.K, dune_max_num=cfg.N, nrmp_max_num=cfg.M, dune_checkpoint=weights_path(cfg.model),
                                      iter_threshold=0.1, max_points=cfg.N))
    batches = WorldBatch(B, pl.robot, lidar, pl.dt)  # the rollout batches' world
    world = WorldBatch(S, pl.robot, lidar, pl.dt)    # the bank's

    def events():
        return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    # warm-up: handles, workspaces and the first launches
    batches.set_scenes(scenes[:B])
    pl.set_initial_paths(scene_paths(scenes[:B]))
    rollout(pl, batches, 3)
    torch.cuda.synchronize()

    # host-driven batches: ceil(S / B) fixed-length rollouts (a short last batch padded with repeats of its first scene)
    nb = (S + B - 1) // B
    e0, e1 = events()
    e0.record()
    for i in range(nb):
        batch = scenes[i * B:(i + 1) * B]
        batch = batch + [batch[0]] * (B - len(batch))
        batches.set_scenes(batch)
        pl.set_initial_paths(scene_paths(batch))
        pl.reset()
        pl.pan.reset_state()
        rollout(pl, batches, T)
    e1.record()
    torch.cuda.synchronize()
    ms_rollout = e0.elapsed_time(e1)

    # continuous episodes
    e0, e1 = events()
    e0.record()
    world.set_episodes(scenes, B, T)
    pl.load_bank(scene_paths(scenes))
    out = run_episodes(pl, world, check_every=args.check_every)
    e1.record()
    torch.cuda.synchronize()
    ms_episodes = e0.elapsed_time(e1)
    end = out["end_step"].cpu().long()
    reason = out["reason"].cpu()
    steps = int(out["steps"])
    useful = int(end.sum())
    waste_rollout = nb * B * T - useful
    waste_episodes = steps * B - useful

    # the advance kernel's device time per step, in a separate run
    from torch.profiler import ProfilerActivity, profile

    world.set_episodes(scenes, B, T)
    pl.load_bank(scene_paths(scenes))
    episode_steps(pl, world, 2)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        episode_steps(pl, world, args.profile_steps)
        torch.cuda.synchronize()
    us = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) for e in prof.key_averages() if "world_advance_kernel" in e.key)
    print(json.dumps(dict(metric="continuous episodes vs fixed-length rollout batches", scene="dyna_obs", behavior="rvo", scenes=S, slots=B,
                          max_steps=T, beams=args.beams, check_every=args.check_every,
                          episodes_per_s=S / (ms_episodes * 1e-3), ms_episodes=ms_episodes, ms_rollout_batches=ms_rollout,
                          rollout_batches=nb, speedup=ms_rollout / ms_episodes, episode_loop_steps=steps,
                          ended_by_flags=int((reason == 1).sum()), ended_by_timeout=int((reason == 2).sum()),
                          mean_end_step=float(end.float().mean()), planner_row_steps_useful=useful,
                          planner_row_steps_after_end_rollout=waste_rollout, planner_row_steps_after_end_episodes=waste_episodes,
                          share_after_end_rollout=waste_rollout / (nb * B * T), share_after_end_episodes=waste_episodes / (steps * B),
                          ms_advance_kernel_per_step=us * 1e-3 / args.profile_steps, **_card())))
    world.close()
    batches.close()
    pl.close()


if __name__ == "__main__":
    main()
