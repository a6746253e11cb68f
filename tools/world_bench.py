"""Times the batched world (csrc/world_kernel.cuh) against the planner it serves, on the device, and prints one JSON line.

    python tools/world_bench.py [--scene dyna_obs|dyna_non_obs|circle_swap] [--behavior constant|rvo] [--envs 4096] [--robots 1]
                                [--beams 1080] [--steps 20] [--warmup 3]

Scenes: seeded dyna_obs (20 moving circles per environment, neupan_b200.world.dyna_obs; the default) or dyna_non_obs (11 moving
obstacles after example/dyna_non_obs: squares, circles and non-convex outlines, neupan_b200.world.dyna_non_obs), with constant-velocity
obstacles (the default) or the examples' reactive ones (--behavior rvo, csrc/world_rvo_kernel.cuh); or circle_swap, --robots K robots
per environment swapping places on a circle (neupan_b200.world.circle_swap; --envs environments x K robots = N planners).  Planner:
PlannerBatch with C4's robot, adjust values and K, the scans decimated to C4's N = 500 points.  Legs, each timed with CUDA events over --steps iterations after
--warmup: the world alone (scan + step), the planner alone (PlannerBatch.forward repeated on the initial states and scans, after a
reset) and the closed-loop step (scan -> PlannerBatch.forward -> step, from the initial scenes after a reset), whose world and planner
parts are also timed separately with events around each call.  The planner-alone leg repeats one input; in the closed loop the
inputs change every step (robots move, some arrive or stop), so the two planner times need not agree.  The card's name and power
limit are read in the same run.  With --behavior rvo, one more closed-loop window of --steps iterations runs under torch.profiler,
which gives the device time of world_rvo_kernel per step and its share of the closed-loop step timed with events.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = (s.strip() for s in out.split(","))
        return dict(gpu=name, power_limit=power, sm_max_clock=clock)
    except Exception as e:  # the timings stand without it, but say why the card is unnamed
        return dict(gpu=None, error=str(e))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scene", choices=("dyna_obs", "dyna_non_obs", "circle_swap"), default="dyna_obs")
    ap.add_argument("--robots", type=int, default=1, help="robots per environment (circle_swap only)")
    ap.add_argument("--behavior", choices=("constant", "rvo"), default="constant")
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--beams", type=int, default=1080)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import math

    import torch

    from helpers import CONFIGS, weights_path
    from neupan_b200 import PlannerBatch, WorldBatch
    from neupan_b200.world import circle_swap, dyna_non_obs, dyna_obs, pack_scenes_ex, scene_paths

    if not torch.cuda.is_available():
        raise SystemExit("world_bench.py needs a CUDA device")
    B, R = args.envs, args.beams
    cfg = CONFIGS["C4"]
    lidar = dict(angle_min=-math.pi, angle_max=math.pi, range_min=0.0, range_max=10.0, number=R)
    if args.scene == "circle_swap":
        scenes = circle_swap(B, robots=args.robots, seed=2024)
    elif args.robots != 1:
        raise SystemExit("--robots needs --scene circle_swap")
    else:
        scenes = (dyna_obs if args.scene == "dyna_obs" else dyna_non_obs)(B, seed=2024, behavior=args.behavior)
    N = B * args.robots
    packed = pack_scenes_ex(scenes)
    n_obs, n_edges = int(packed[0][-1]), int(packed[2][-1])
    n_circles = int((packed[2][1:] == packed[2][:-1]).sum())
    pl = PlannerBatch(N, cfg.T, cfg.dt, 4.0, robot_kwargs=cfg.robot_kwargs, adjust_kwargs=dict(cfg.adjust),
                      pan_kwargs=dict(iter_num=cfg.K, dune_max_num=cfg.N, nrmp_max_num=cfg.M, dune_checkpoint=weights_path(cfg.model),
                                      iter_threshold=0.0, max_points=cfg.N))
    pl.set_initial_paths(scene_paths(scenes))
    world = WorldBatch(B, pl.robot, lidar, pl.dt)
    world.set_scenes(scenes)
    zero = torch.zeros(N, 2, device="cuda")
    ranges0, vel0, scan0 = world.scan()
    states0 = world.states

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    def world_only():
        world.scan()
        world.step(zero)

    def planner_only():
        pl.forward(states0, ranges0, scan0, scan_offset=world.scan_offset, scan_velocity=vel0)

    split = []  # per closed-loop step: events before the scan, after it, after the planner, after the step

    def closed_loop():
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        r, v, s = world.scan()
        ev[1].record()
        a, _ = pl.forward(world.states, r, s, scan_offset=world.scan_offset, scan_velocity=v)
        ev[2].record()
        world.step(a)
        ev[3].record()
        split.append(ev)

    ms_scan = timed(world.scan)
    ms_world = timed(world_only)
    pl.reset()
    ms_planner = timed(planner_only)
    world.set_scenes(scenes)
    pl.reset()
    ms_loop = timed(closed_loop)
    timed_steps = split[-args.steps:]  # the events of the timed window (all recorded and synchronised by timed())
    ms_loop_world = sum(e[0].elapsed_time(e[1]) + e[2].elapsed_time(e[3]) for e in timed_steps) / args.steps
    ms_loop_planner = sum(e[1].elapsed_time(e[2]) for e in timed_steps) / args.steps
    rvo = {}
    if args.behavior == "rvo":  # device time of the reactive obstacles' kernel inside the closed loop
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                closed_loop()
            torch.cuda.synchronize()
        us = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) for e in prof.key_averages() if "world_rvo_kernel" in e.key)
        rvo = dict(ms_rvo_kernel=us * 1e-3 / args.steps, rvo_share_of_closed_loop=us * 1e-3 / args.steps / ms_loop)
    tests = args.robots * R * (n_circles + n_edges)  # ray-obstacle tests of one scan: every beam against every circle and polygon edge
    print(json.dumps(dict(metric="batched world: scan + step vs PlannerBatch.forward", scene=args.scene, behavior=args.behavior, envs=B,
                          robots_per_env=args.robots, planners=N, beams=R,
                          obstacles_per_env=n_obs / B, circles_per_env=n_circles / B, edges_per_env=n_edges / B,
                          steps=args.steps, warmup=args.warmup, ms_scan=ms_scan, ms_world_scan_step=ms_world, ms_planner_forward=ms_planner,
                          ms_closed_loop_step=ms_loop, ms_closed_loop_world=ms_loop_world, ms_closed_loop_planner=ms_loop_planner,
                          world_share_of_closed_loop=ms_loop_world / ms_loop,
                          ray_obstacle_tests_per_s=tests / (ms_scan * 1e-3), **rvo, **_card())))
    world.close()
    pl.close()


if __name__ == "__main__":
    main()
