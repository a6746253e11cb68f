"""The screening pass for clouds of <= 512 points (dune_screen_warp_kernel, csrc/dune_screen_mma_kernel.cuh): one warp per
(environment, step) item, CTAs persistent over environments with the next environment's cloud staged behind the current one.  Each
case compares the screening pipeline (dune_kernel = 4) with the full kernel (2) bit for bit, with step-0 reuse on and off, at the
shapes where that layout has edges: horizons whose item count does not divide among the CTA's warps, batches smaller than the grid,
ragged and inactive environments in one CTA, the cloud sizes around the tile and kernel boundaries, and items whose tiles partly
leave the distance table."""
import dataclasses

import numpy as np
import pytest
import torch

from gpu_helpers import make_pan, run_pan, to_cuda
from helpers import CONFIGS, make_inputs

pytestmark = pytest.mark.gpu


def _outputs(pan, t, counts=None):
    with torch.no_grad():
        S, U, D = pan(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"], num_points=counts)
    sel = {k: v.cpu().numpy() for k, v in pan.read_selection().items()}
    return S.cpu().numpy(), U.cpu().numpy(), D.cpu().numpy(), pan.min_distance.cpu().numpy(), sel


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


def _compare(cfg, inp, K, N, skip_t0, counts=None, **kw):
    """Full kernel vs screening pipeline on the same inputs; returns the screening handle's statistics."""
    t = to_cuda(inp)
    B = inp["nom_s"].shape[0]
    c = None if counts is None else torch.tensor(counts, dtype=torch.int32).cuda()
    outs, pans = [], []
    for dk in (2, 4):
        pan = make_pan(cfg, K=K, N=N, max_envs=B, dune_kernel=dk, dune_skip_t0=skip_t0, **kw)
        outs.append(_outputs(pan, t, c))
        pans.append(pan)
    _assert_equal(*outs)
    return pans[1].screen_stats()


@pytest.mark.parametrize("skip_t0", [0, 1])
@pytest.mark.parametrize("T", [5, 15])
def test_horizons_not_a_multiple_of_the_warps(T, skip_t0):
    cfg = dataclasses.replace(CONFIGS["C4"], T=T)
    inp = make_inputs(cfg, B=9, N=400, scene="obstacles")
    st = _compare(cfg, inp, 3, 400, skip_t0)
    assert st["screened_items"] > 0


@pytest.mark.parametrize("skip_t0", [0, 1])
@pytest.mark.parametrize("B", [1, 3])
def test_batches_smaller_than_the_grid(B, skip_t0):
    cfg = CONFIGS["C4"]
    _compare(cfg, make_inputs(cfg, B=B, scene="annulus"), 3, cfg.N, skip_t0)


@pytest.mark.parametrize("skip_t0", [0, 1])
def test_ragged_and_inactive_environments_within_one_cta(skip_t0):
    """B = 2000 at most a few hundred CTAs: every CTA runs several environments in a row, so consecutive environments of one CTA
    have different counts (ragged, <= 32, 0) and the stop criterion switches some of them off between PAN iterations."""
    cfg = CONFIGS["C4"]
    B, N = 2000, 500
    inp = make_inputs(cfg, B=B, N=N, scene="obstacles")
    counts = np.array([500, 0, 37, 32, 499, 5, 33, 256, 480, 1, 511, 64, 300], dtype=np.int32)
    counts = np.resize(counts, B)
    _compare(cfg, inp, 3, N, skip_t0, counts=counts.tolist())
    _compare(cfg, inp, 6, N, skip_t0, counts=counts.tolist(), iter_threshold=0.1)


@pytest.mark.parametrize("skip_t0", [0, 1])
@pytest.mark.parametrize("N", [33, 511, 512, 513])
def test_cloud_sizes_at_the_tile_and_kernel_boundaries(N, skip_t0):
    cfg = CONFIGS["C4"]
    _compare(cfg, make_inputs(cfg, B=12, N=N, scene="obstacles"), 3, N, skip_t0)


@pytest.mark.parametrize("skip_t0", [0, 1])
def test_items_with_tiles_inside_and_outside_the_table(skip_t0):
    """Points scattered up to twice the table's half-width (16.4 m) from the robot: most items have tiles that the table covers
    completely next to tiles with a point outside it, which run the network.  Also the acker checkpoint, which has no table."""
    cfg = CONFIGS["C4"]
    inp = make_inputs(cfg, B=16, N=500, scene="annulus")
    rng = np.random.default_rng(7)
    nom = inp["nom_s"]
    pts = inp["points"].copy()
    for b in range(pts.shape[0]):
        far = rng.random(pts.shape[2]) < 0.03
        ang = rng.uniform(0, 2 * np.pi, far.sum())
        r = rng.uniform(17.0, 30.0, far.sum())
        pts[b, 0, far] = nom[b, 0, 0] + r * np.cos(ang)
        pts[b, 1, far] = nom[b, 1, 0] + r * np.sin(ang)
    inp = dict(inp, points=pts.astype(inp["points"].dtype))
    st = _compare(cfg, inp, 3, 500, skip_t0)
    assert st["screened_items"] > 0
    cfg2 = CONFIGS["C2"]
    _compare(cfg2, make_inputs(cfg2, B=12, N=300, scene="obstacles"), 3, 300, skip_t0)


@pytest.mark.parametrize("skip_t0", [0, 1])
def test_statistics_count_every_screened_item_once(skip_t0):
    """screen_stats is collected per CTA and flushed at the end of the launch: every item with n > 32 is either screened (with M to
    32 candidates) or flagged for the exact kernel, exactly once per launch."""
    cfg = CONFIGS["C4"]
    B, K = 1500, 3
    inp = make_inputs(cfg, B=B, scene="annulus")
    pan = make_pan(cfg, K=K, max_envs=B, dune_kernel=4, dune_skip_t0=skip_t0)
    pan.screen_stats()
    run_pan(pan, inp)
    st = pan.screen_stats()
    T1 = cfg.T + 1
    items = B * T1 + (K - 1) * B * (cfg.T if skip_t0 else T1)
    assert st["screened_items"] <= items <= st["screened_items"] + st["exact_items"], st
    assert cfg.M * st["screened_items"] <= st["candidates"] <= 32 * st["screened_items"], st
