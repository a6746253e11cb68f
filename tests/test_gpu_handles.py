"""Device memory of the C handles (nb_buffer_count): every handle gives back all it allocated when it is destroyed, after regrowths,
replaced state and dropped state alike; a world that went through every set call holds what a fresh world with the same scenes
holds; and a nb_pan_create that fails on an allocation leaves nothing behind and the next handle computes as before."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

from gpu_helpers import make_pan, run_pan, to_cuda
from helpers import CONFIGS, make_inputs
from neupan_b200 import InitialPathBatch, WorldBatch, _lib
from neupan_b200.blocks.dune_train import DUNETrain
from neupan_b200.blocks.obs_point_net import ObsPointNet
from neupan_b200.world import _host_ptrs, line_path, maze, pack_behaviors, pack_fleet, pack_map_contact, pack_maps, pack_scenes_ex
from test_gpu_world import LIDAR
from test_gpu_world_mixed import _robot

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def no_collector():
    """Handles of earlier tests that sit in reference cycles must not be destroyed in the middle of a count."""
    gc.collect()
    gc.disable()
    yield
    gc.enable()


def count():
    torch.cuda.synchronize()
    return _lib.load().nb_buffer_count()


def test_pan_handles_give_back_every_buffer():
    """C4 with DUNE (screening pipeline, distance table and calibration temporaries), a no-obstacle handle, a differentiable handle
    whose iter_num grows between two forwards (the adjoint records are replaced), and the host entry point with a growing B (the
    staging buffers grow)."""
    cfg = CONFIGS["C4"]
    inp = make_inputs(cfg, B=4, scene="obstacles")
    t = to_cuda(inp)
    for kw in (dict(), dict(M=0)):
        n0 = count()
        pan = make_pan(cfg, max_envs=4, **kw)
        with torch.no_grad():
            pan(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"])
        assert count() > n0
        pan.close()
        assert count() == n0, kw

    n0 = count()
    pan = make_pan(cfg, K=2, max_envs=4)
    with torch.enable_grad():  # the suite runs inference tests under no_grad
        for K in (2, 4):
            pan.iter_num = K
            S, U, D = pan(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"])
            assert S.requires_grad
            (S.sum() + U.sum()).backward()
    pan.close()
    assert count() == n0

    n0 = count()
    pan = make_pan(cfg, max_envs=16)
    for B in (2, 16):
        S, U, D, md = run_pan(pan, make_inputs(cfg, B=B, scene="obstacles"), cuda=False)
        assert S.shape[0] == B
    pan.close()
    assert count() == n0


def test_world_set_calls_hold_what_a_fresh_world_holds():
    """set_scenes -> behaviours -> fleet -> maps with contact -> episodes -> set_scenes with the first scenes holds what a fresh world
    holds after that first set_scenes; both give back everything when destroyed."""
    B = 8
    rb = _robot("diff")
    scenes = maze(B, seed=4, movers=4, behavior="rvo")
    assert pack_map_contact(scenes).all()
    packed, beh, rows = pack_scenes_ex(scenes), pack_behaviors(scenes), pack_fleet(scenes)
    maps = pack_maps(scenes)
    contact = pack_map_contact(scenes)
    lib = _lib.load()
    n0 = count()
    fresh = WorldBatch(B, rb, LIDAR | dict(number=90), 0.1)
    with torch.cuda.device(fresh.device):
        _lib.check(lib.nb_world_set_scenes_ex(fresh._handle, B, *_host_ptrs(packed)))
        held = count() - n0
        n1 = count()
        w = WorldBatch(B, rb, LIDAR | dict(number=90), 0.1)
        h = w._handle
        _lib.check(lib.nb_world_set_scenes_ex(h, B, *_host_ptrs(packed)))
        _lib.check(lib.nb_world_set_behaviors(h, B, C.c_void_p(beh.ctypes.data), C.c_uint64(3)))
        _lib.check(lib.nb_world_set_fleet(h, B, 1, C.c_void_p(rows.ctypes.data)))
        _lib.check(lib.nb_world_set_maps(h, len(maps[0]), maps[0], C.c_void_p(maps[1].ctypes.data), C.c_void_p(maps[2].ctypes.data),
                                         C.c_double(1.0)))
        _lib.check(lib.nb_world_set_map_contact(h, B, C.c_void_p(contact.ctypes.data)))
        _lib.check(lib.nb_world_set_episodes(h, B // 2, 50))
        assert count() - n1 > held
        _lib.check(lib.nb_world_set_scenes_ex(h, B, *_host_ptrs(packed)))
    assert count() - n1 == held
    fresh.close()
    w.close()
    assert count() == n0


def test_ipath_and_training_handles_give_back_every_buffer():
    """set_paths twice, the second time with more environments and points; train_one_epoch with a growing batch count."""
    n0 = count()
    ipb = InitialPathBatch(10, 0.1, "diff", max_envs=6)
    ipb.set_initial_paths([line_path((0, 0), (5, 1)) for _ in range(2)])
    ipb.set_initial_paths([line_path((0, b), (20, b)) for b in range(6)])
    ipb.close()
    assert count() == n0

    rb = CONFIGS["C1"].make_robot()
    G, h = np.asarray(rb.G, np.float32), np.asarray(rb.h, np.float32).reshape(-1)
    torch.manual_seed(0)
    np.random.seed(1)
    n0 = count()
    tr = DUNETrain(ObsPointNet(2, G.shape[0]), G, h, "/tmp/unused", backend="native")
    for n in (300, 2000):
        tr.train_one_epoch(tr.generate_data_set(n, [-8, -8, 8, 8]), 256)
    tr.close()
    assert count() == n0


def test_failed_pan_create_leaves_nothing_behind():
    """max_envs = 2^30: the first large request (cand_idx, about 1.5 TB) exceeds the device; cudaMalloc refuses it, nb_pan_create
    returns NB_ERR_CUDA with the out-pointer NULL and nothing held, and a handle created afterwards computes bitwise what one created
    before the failure did."""
    cfg = CONFIGS["C4"]
    inp = make_inputs(cfg, B=3, scene="obstacles")
    before = make_pan(cfg, max_envs=3)
    ref = run_pan(before, inp)
    before.close()

    big = make_pan(cfg, max_envs=3)
    lib = big._ensure_handle(3, cfg.N)  # a working handle of the same PAN, for its configuration and weights
    big.close()
    ccfg = big._config(2**30, cfg.N)
    w = _lib.pack_weights(big.dune_layer.model.state_dict())
    G = np.ascontiguousarray(np.asarray(big.robot.G), dtype=np.float32)
    h = np.ascontiguousarray(np.asarray(big.robot.h), dtype=np.float32).reshape(-1)
    n0 = count()
    out = C.c_void_p(1)
    rc = lib.nb_pan_create(C.byref(ccfg), w.ctypes.data, w.size, G.ctypes.data, h.ctypes.data, C.byref(out))
    assert rc == _lib.NB_ERR_CUDA, lib.nb_last_error()
    assert out.value is None
    assert count() == n0

    after = make_pan(cfg, max_envs=3)
    got = run_pan(after, inp)
    after.close()
    assert all(np.array_equal(a, b) for a, b in zip(ref, got))
