"""DUNE with screening (NB_OPT_DUNE_KERNEL = 4, csrc/dune_screen_kernel.cuh): a single-pass fp16 interval pass selects the <= 32 points
per (environment, step) that can be among the M closest, the exact network runs only on them.  The contract is equality with the
full kernel (variant 2) BIT FOR BIT -- selections, mu, lam, distances, and therefore the whole PAN output -- plus a measured margin
between the screening error and the bound c_mu the intervals are built with."""
import os

import numpy as np
import pytest
import torch

from gpu_helpers import make_pan, record, run_pan, to_cuda
from helpers import CONFIGS, make_inputs

pytestmark = pytest.mark.gpu


def _pair(cfg, inp, K, **kw):
    out = []
    for dk in (2, 4):
        pan = make_pan(cfg, K=K, max_envs=inp["nom_s"].shape[0], dune_kernel=dk, **kw)
        S, U, D, md = run_pan(pan, inp)
        sel = {k: v.cpu().numpy() for k, v in pan.read_selection().items()}
        out.append((S, U, D, md, sel, pan))
    return out


def _assert_equal(a, b):
    for x, y in zip(a[:4], b[:4]):
        assert np.array_equal(x, y)
    cnt = a[4]["count"]
    assert np.array_equal(cnt, b[4]["count"])
    M = a[4]["distance"].shape[-1]
    live = np.arange(M)[None, None, :] < cnt[:, None, None]  # rows beyond min(n, M) are never written
    for k in ("mu", "lam", "points", "distance"):
        x, y = a[4][k], b[4][k]
        m = live if x.ndim == 3 else live[..., None]
        assert np.array_equal(np.where(m, x, 0), np.where(m, y, 0)), k


@pytest.mark.parametrize("cname", ["C1", "C2", "C3", "C4", "C5"])
@pytest.mark.parametrize("scene", ["annulus", "obstacles"])
def test_screened_equals_full_kernel_bitwise(cname, scene):
    cfg = CONFIGS[cname]
    B = 12 if cname != "C5" else 6
    inp = make_inputs(cfg, B=B, scene=scene)
    for K in (1, 3):
        full, scr = _pair(cfg, inp, K)
        _assert_equal(full, scr)
    st = scr[5].screen_stats()
    record("dune_screen", config=cname, scene=scene, **st, candidates_per_item=st["candidates"] / max(1, st["screened_items"]),
           exact_fraction=st["exact_items"] / max(1, st["exact_items"] + st["screened_items"]))
    assert st["max_error_ratio"] < st["c_mu"], st  # the error measured on every refined candidate stays inside the radius the intervals assume
    assert st["screened_items"] > 0


@pytest.mark.parametrize("screen_mma,skip_t0", [(0, 0), (0, 1), (1, 0)])
@pytest.mark.parametrize("cname", ["C2", "C4", "C5"])
def test_screen_shapes_and_step0_reuse_equal_full_kernel_bitwise(cname, screen_mma, skip_t0):
    """The non-default combinations of NB_OPT_DUNE_SCREEN_MMA (screening pass on wgmma / mma.sync) and NB_OPT_DUNE_SKIP_T0 (step-0
    items of PAN iterations k > 0 re-evaluated / kept): same bits as the full kernel, like the defaults in the tests above."""
    cfg = CONFIGS[cname]
    inp = make_inputs(cfg, B=12 if cname != "C5" else 6, scene="obstacles" if cname == "C2" else "annulus")
    full, scr = _pair(cfg, inp, 3, dune_screen_mma=screen_mma, dune_skip_t0=skip_t0)
    _assert_equal(full, scr)
    assert scr[5].screen_stats()["screened_items"] > 0


def test_full_size_c4_bitwise_and_statistics():
    cfg = CONFIGS["C4"]
    inp = make_inputs(cfg, B=4096)
    full, scr = _pair(cfg, inp, cfg.K)
    _assert_equal(full, scr)
    st = scr[5].screen_stats()
    record("dune_screen_c4_full", **st, candidates_per_item=st["candidates"] / max(1, st["screened_items"]),
           exact_fraction=st["exact_items"] / max(1, st["exact_items"] + st["screened_items"]))
    assert st["max_error_ratio"] < st["c_mu"]
    assert st["exact_items"] < 0.05 * (st["exact_items"] + st["screened_items"])


def test_small_ragged_and_stopped_environments():
    cfg = CONFIGS["C4"]
    # N <= 32 (no screening), N just above, ragged counts incl. 0 and < M
    for N in (8, 33, 40, 200):
        inp = make_inputs(cfg, B=5, N=N, scene="obstacles")
        full, scr = _pair(cfg, inp, 2, N=N)
        _assert_equal(full, scr)
    inp = make_inputs(cfg, B=6, N=300, scene="obstacles")
    counts = torch.tensor([300, 0, 5, 33, 150, 32], dtype=torch.int32).cuda()
    t = to_cuda(inp)
    outs = []
    for dk in (2, 4):
        pan = make_pan(cfg, K=2, N=300, max_envs=6, dune_kernel=dk)
        S, U, D = pan(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"], num_points=counts)
        outs.append((S.cpu().numpy(), U.cpu().numpy(), D.cpu().numpy(), pan.min_distance.cpu().numpy()))
    for x, y in zip(*outs):
        assert np.array_equal(x, y)
    # the stop criterion switches environments off between iterations: their items are skipped by all three kernels
    cfg5 = CONFIGS["C5"]
    inp = make_inputs(cfg5, B=8, scene="obstacles")
    a, b = _pair(cfg5, inp, 6, iter_threshold=0.1)
    _assert_equal(a, b)
    assert np.array_equal(a[5].iterations.cpu().numpy(), b[5].iterations.cpu().numpy())


def test_items_the_screen_cannot_narrow_down_take_the_exact_path():
    """A huge bound makes every interval overlap: all items are flagged and evaluated by the full kernel."""
    cfg = CONFIGS["C2"]
    inp = make_inputs(cfg, B=6, scene="annulus")
    os.environ["NB_SCREEN_CMU"] = "10.0"
    try:
        full, scr = _pair(cfg, inp, 2)
    finally:
        del os.environ["NB_SCREEN_CMU"]
    _assert_equal(full, scr)
    st = scr[5].screen_stats()
    assert st["screened_items"] == 0 and st["exact_items"] > 0
