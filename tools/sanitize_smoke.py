"""Small runs covering every kernel path, for compute-sanitizer (memcheck / racecheck / initcheck):
    compute-sanitizer --tool memcheck python tools/sanitize_smoke.py"""
import os, sys
sys.path.insert(0, os.getcwd()); sys.path.insert(0, "tests")
import numpy as np, torch
from gpu_helpers import make_pan, run_pan, to_cuda
from helpers import CONFIGS, make_inputs
SECTIONS = os.environ.get("NB_SMOKE_SECTIONS", "variants,screen,adjoint,train,world").split(",")
# N = 300: two slots, then a pass with one; N = 600: keys in shared memory (n > 512)
for cname, B, N in (("C4", 6, 70), ("C5", 3, 40), ("C2", 5, 33), ("C4", 3, 300), ("C3", 2, 600)) if "variants" in SECTIONS else ():
    cfg = CONFIGS[cname]
    inp = make_inputs(cfg, B=B, N=N, scene="obstacles")
    pan = make_pan(cfg, K=2, N=N, max_envs=B, dune_kernel=2, nrmp_warm=1)
    S, U, D, md = run_pan(pan, inp)
    assert np.isfinite(S).all() and (pan.status.cpu().numpy() == 0).all()
    pan.close()
# round 2: the screening pipeline (both screening kernels, step-0 reuse, paired refine, exact remainder), the stop criterion as its own
# kernel (B >= 256), sub-batches on internal streams (B >= 128) and the chunked upload (nb_pan_forward_h2d / _host)
if "screen" in SECTIONS:
    for cname, B, N, K in (("C4", 7, 70, 3), ("C4", 3, 300, 2), ("C3", 2, 600, 2), ("C2", 260, 40, 3), ("C5", 130, 36, 2)):
        cfg = CONFIGS[cname]
        inp = make_inputs(cfg, B=B, N=N, scene="obstacles")
        for mma, skip in ((1, 1), (0, 1), (1, 0)):
            pan = make_pan(cfg, K=K, N=N, max_envs=B, dune_kernel=4, dune_screen_mma=mma, dune_skip_t0=skip, iter_threshold=0.05 if B > 100 else 0.0)
            S, U, D, md = run_pan(pan, inp)
            assert np.isfinite(S).all() and (pan.status.cpu().numpy() == 0).all()
            if B > 100 and mma and skip:
                pin = {k: (None if v is None else torch.from_numpy(np.ascontiguousarray(v)).pin_memory()) for k, v in inp.items()}
                with torch.no_grad():
                    for dev_out in (True, False):
                        out = pan(pin["nom_s"], pin["nom_u"], pin["ref_s"], pin["ref_us"], pin["points"], pin["velocities"], device_out=dev_out)
                        torch.cuda.synchronize()
                        assert torch.isfinite(out[0]).all()
            pan.close()
# persistent NRMP warps (more environments than resident warps is not needed: the counter path is taken when grid > resident) + adjoint
for cname, B in (("C4", 5), ("C5", 3), ("C1", 2)) if "adjoint" in SECTIONS else ():
    cfg = CONFIGS[cname]
    inp = make_inputs(cfg, B=B, N=50, scene="obstacles")
    pan = make_pan(cfg, K=2, N=50, max_envs=B)
    t = to_cuda(inp)
    S, U, D = pan(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"])
    (S.sum() + U.sum() + D.sum()).backward()
    assert all(torch.isfinite(p.grad).all() for p in pan.nrmp_layer.adjust_parameters)
    pan.close()
# training kernels (ragged last batch)
from neupan_b200.blocks.dune_train import DUNETrain
from neupan_b200.blocks.obs_point_net import ObsPointNet
for cname in ("C1", "C5") if "train" in SECTIONS else ():
    rb = CONFIGS[cname].make_robot()
    G, h = np.asarray(rb.G, np.float32), np.asarray(rb.h, np.float32).reshape(-1)
    tr = DUNETrain(ObsPointNet(2, G.shape[0]), G, h, "/tmp/unused", backend="native")
    data = tr.generate_data_set(600, [-25, -25, 25, 25])
    for _ in range(2):
        losses = tr.train_one_epoch(data, 256, False)
    tr.train_one_epoch(data, 256, True)
    assert np.isfinite(losses).all()
    tr.sync_model(); tr.close()
# the batched world with reactive obstacles: world_scan_kernel, world_rvo_kernel (goal draws, the robot as a neighbour of an obstacle
# placed on its path) and world_step_kernel (every K; here one robot per environment, a one-warp CTA)
if "world" in SECTIONS:
    from neupan_b200 import WorldBatch
    from neupan_b200.world import dyna_non_obs, dyna_obs
    rb = CONFIGS["C4"].make_robot()
    lidar = dict(angle_min=-np.pi / 2, angle_max=np.pi / 2, range_min=0.0, range_max=10.0, number=100)
    for builder in (dyna_obs, dyna_non_obs):
        scenes = builder(6, seed=1, behavior="rvo")
        scenes[0]["obstacles"].append(dict(center=(12.0, scenes[0]["start"][1]), radius=0.3, behavior=dict(name="rvo", vxmax=0.5, vymax=0.5,
                                                                                                       goal=(20.0, 20.0))))
        w = WorldBatch(6, rb, lidar, 0.1)
        w.set_scenes(scenes, seed=3)
        for _ in range(30):
            w.scan()
            w.step(torch.full((6, 2), 0.5, device="cuda"))
        g, d = w.goals()
        torch.cuda.synchronize()
        assert torch.isfinite(w.obstacles()).all() and torch.isfinite(g).all()
        w.close()
    # a mixed fleet: C4's diff robot, C2's car and C5's trapezoid, six robots per environment, with reactive obstacles among them
    from neupan_b200.world import mixed_swap
    kinds = [CONFIGS[c].make_robot() for c in ("C4", "C2", "C5")]
    scenes = mixed_swap(6, robots=6, seed=1, circles=3)
    for sc in scenes:
        sc["obstacles"] = [dict(ob, behavior=dict(name="rvo", vxmax=0.5, vymax=0.5, wander=True)) for ob in sc["obstacles"]]
    w = WorldBatch(6, kinds, lidar, 0.1)
    w.set_scenes(scenes, seed=3)
    for _ in range(30):
        w.scan()
        w.step(torch.full((36, 2), 0.5, device="cuda"))
    torch.cuda.synchronize()
    assert torch.isfinite(w.states).all() and torch.isfinite(w.obstacles()).all()
    w.close()
    # occupancy maps: the map instantiations of world_scan_kernel and world_step_kernel, a maze in four environments and a map-free
    # environment beside them
    from neupan_b200.world import maze
    scenes = maze(5, cells=(3, 3), seed=1, layouts=2) + dyna_obs(1, seed=1)
    w = WorldBatch(6, rb, lidar, 0.1)
    w.set_scenes(scenes)
    for _ in range(30):
        r, _, _, hit = w.scan(hit=True)
        w.step(torch.full((6, 2), 0.5, device="cuda"))
    torch.cuda.synchronize()
    assert torch.isfinite(w.states).all() and (hit[:5] == 1).any()  # no obstacles, K = 1: the map is index 1
    w.close()
    # maps that block obstacles: the blocking step and rvo instantiations, constant and reactive movers in mazes
    for behavior in ("constant", "rvo"):
        w = WorldBatch(4, rb, lidar, 0.1)
        w.set_scenes(maze(4, cells=(4, 4), seed=1, layouts=2, movers=6, behavior=behavior))
        for _ in range(30):
            w.scan()
            w.step(torch.full((4, 2), 0.5, device="cuda"))
        torch.cuda.synchronize()
        assert torch.isfinite(w.obstacles()).all() and (w.map_bounces() >= 0).all()
        w.close()
    # obstacle contact: the contact kernel and the step without obstacle motion, plain and over blocking maps, constant and reactive
    from neupan_b200.world import dyna_non_obs
    for scenes in (dyna_non_obs(3, seed=1, behavior="rvo", contact=True) + dyna_obs(1, seed=1),
                   maze(4, cells=(4, 4), seed=1, layouts=2, movers=6, behavior="rvo", contact=True)):
        w = WorldBatch(4, rb, lidar, 0.1)
        w.set_scenes(scenes)
        for _ in range(30):
            w.scan()
            w.step(torch.full((4, 2), 0.5, device="cuda"))
        torch.cuda.synchronize()
        assert torch.isfinite(w.obstacles()).all() and (w.obstacle_bounces() >= 0).all()
        w.close()
    # continuous episodes: the episode instantiations of the scan, rvo and step kernels, the advance and slot gather kernels, and the
    # per-slot ipath and PAN calls, through run_episodes over a bank of 7 scenes in 3 slots (some slots go idle); then a maze bank
    # with its map through 2 slots, stepped until every slot is idle
    from helpers import weights_path
    from neupan_b200 import PlannerBatch, run_episodes
    from neupan_b200.world import scene_paths
    c4 = CONFIGS["C4"]
    pl = PlannerBatch(3, c4.T, c4.dt, 4.0, robot_kwargs=c4.robot_kwargs, adjust_kwargs=dict(c4.adjust),
                      pan_kwargs=dict(iter_num=2, dune_max_num=100, nrmp_max_num=c4.M, dune_checkpoint=weights_path(c4.model), iter_threshold=0.1,
                                      max_points=100))
    scenes = dyna_obs(7, seed=1, behavior="rvo")
    w = WorldBatch(7, rb, lidar, 0.1)
    w.set_episodes(scenes, 3, 6, seed=3)
    pl.load_bank(scene_paths(scenes))
    out = run_episodes(pl, w, check_every=4)
    assert (out["reason"] > 0).all()
    pl.close()
    w.close()
    scenes = maze(5, cells=(3, 3), seed=1, layouts=2)
    w = WorldBatch(5, rb, lidar, 0.1)
    w.set_episodes(scenes, 2, 3)
    for _ in range(10):
        w.scan(hit=True)
        w.step(torch.full((2, 2), 0.5, device="cuda"))
    torch.cuda.synchronize()
    assert int(w.finished().item()) == 5 and torch.isfinite(w.states).all()
    w.close()
torch.cuda.synchronize()
print("sanitize smoke ok")
