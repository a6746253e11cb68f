"""The two-level table path of the one-warp-per-item screen (dune_screen_warp_kernel, csrc/dune_screen_mma_kernel.cuh): an item whose
points all lie in the distance table is bounded from the coarse bound table first, and only the points that survive gather their fine
cell.  Its candidates are those of the one-level path by construction, so every case runs a handle created with NB_SCREEN_COARSE=0
(every item on the one-level path) against the default handle and asks for the same outputs, selection and screen statistics bit
for bit."""
import numpy as np
import pytest
import torch

from gpu_helpers import make_pan, record, to_cuda
from helpers import CONFIGS, make_inputs

pytestmark = pytest.mark.gpu

SAME_STATS = ("max_error_ratio", "exact_items", "candidates", "screened_items")


def _run(monkeypatch, coarse, cfg, inp, K, skip_t0, counts=None, **kw):
    monkeypatch.setenv("NB_SCREEN_COARSE", str(coarse))  # read when the handle is created, at the first forward
    B, N = inp["points"].shape[0], inp["points"].shape[2]
    pan = make_pan(cfg, K=K, N=N, max_envs=B, dune_skip_t0=skip_t0, **kw)
    t = to_cuda(inp)
    c = None if counts is None else torch.tensor(counts, dtype=torch.int32).cuda()
    with torch.no_grad():
        S, U, D = pan(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"], num_points=c)
    monkeypatch.delenv("NB_SCREEN_COARSE")
    sel = {k: v.cpu().numpy() for k, v in pan.read_selection().items()}
    out = (S.cpu().numpy(), U.cpu().numpy(), D.cpu().numpy(), pan.min_distance.cpu().numpy(), sel)
    return out, pan.screen_stats()


def _compare(monkeypatch, cfg, inp, K, skip_t0, counts=None, **kw):
    ref, st0 = _run(monkeypatch, 0, cfg, inp, K, skip_t0, counts, **kw)
    got, st1 = _run(monkeypatch, 1, cfg, inp, K, skip_t0, counts, **kw)
    for x, y in zip(ref[:4], got[:4]):
        assert np.array_equal(x, y)
    cnt = ref[4]["count"]
    assert np.array_equal(cnt, got[4]["count"])
    live = np.arange(ref[4]["distance"].shape[-1])[None, None, :] < cnt[:, None, None]  # rows beyond min(n, M) are never written
    for k in ("mu", "lam", "points", "distance"):
        m = live if ref[4][k].ndim == 3 else live[..., None]
        assert np.array_equal(np.where(m, ref[4][k], 0), np.where(m, got[4][k], 0)), k
    for k in SAME_STATS:
        assert st0[k] == st1[k], k
    assert st0["coarse_survivors"] == 0 and st0["coarse_fallback_items"] == 0
    return st1


@pytest.mark.parametrize("skip_t0", [0, 1])
@pytest.mark.parametrize("scene", ["annulus", "obstacles"])
@pytest.mark.parametrize("cname", ["C1", "C4"])
def test_two_level_path_equals_one_level_path(monkeypatch, cname, scene, skip_t0):
    cfg = CONFIGS[cname]
    st = _compare(monkeypatch, cfg, make_inputs(cfg, B=24, scene=scene), 3, skip_t0)
    if cfg.N > 32:
        assert st["coarse_survivors"] > 0


@pytest.mark.parametrize("skip_t0", [0, 1])
def test_ragged_and_inactive_environments(monkeypatch, skip_t0):
    cfg = CONFIGS["C4"]
    B, N = 600, 500
    counts = np.resize(np.array([500, 0, 37, 32, 499, 5, 33, 256, 480, 1, 511, 64, 300], dtype=np.int32), B)
    counts = np.minimum(counts, N)
    inp = make_inputs(cfg, B=B, N=N, scene="obstacles")
    _compare(monkeypatch, cfg, inp, 3, skip_t0, counts=counts.tolist())
    _compare(monkeypatch, cfg, inp, 6, skip_t0, counts=counts.tolist(), iter_threshold=0.1)


@pytest.mark.parametrize("skip_t0", [0, 1])
def test_points_outside_the_table_and_crowded_items_take_the_one_level_path(monkeypatch, skip_t0):
    """Some environments have points beyond the table (17-30 m away); others pack 300 points within 0.3 m of the
    robot's path, more survivors than the two-level path holds.  Both kinds take the one-level path; the rest take the two-level one."""
    cfg = CONFIGS["C4"]
    B, N = 24, 500
    inp = make_inputs(cfg, B=B, N=N, scene="annulus")
    rng = np.random.default_rng(11)
    nom, pts = inp["nom_s"], inp["points"].copy()
    for b in range(B):
        if b % 3 == 0:
            far = rng.random(N) < 0.03
            ang, r = rng.uniform(0, 2 * np.pi, far.sum()), rng.uniform(17.0, 30.0, far.sum())
            pts[b, 0, far] = nom[b, 0, 0] + r * np.cos(ang)
            pts[b, 1, far] = nom[b, 1, 0] + r * np.sin(ang)
        elif b % 3 == 1:
            k = rng.integers(0, nom.shape[2], 300)
            ang, r = rng.uniform(0, 2 * np.pi, 300), rng.uniform(0.0, 0.3, 300)
            pts[b, 0, :300] = nom[b, 0, k] + r * np.cos(ang)
            pts[b, 1, :300] = nom[b, 1, k] + r * np.sin(ang)
    inp = dict(inp, points=pts.astype(inp["points"].dtype))
    st = _compare(monkeypatch, cfg, inp, 3, skip_t0)
    assert st["coarse_fallback_items"] > 0 and st["coarse_survivors"] > 0


def test_full_size_c4_mostly_takes_the_two_level_path(monkeypatch):
    cfg = CONFIGS["C4"]
    st = _compare(monkeypatch, cfg, make_inputs(cfg, B=cfg.B, scene="annulus"), cfg.K, 1)
    two_level = st["screened_items"] + st["exact_items"] - st["coarse_fallback_items"]
    record("dune_screen_coarse", config="C4", B=cfg.B, survivors_per_item=st["coarse_survivors"] / max(two_level, 1),
           fallback_fraction=st["coarse_fallback_items"] / max(st["screened_items"] + st["exact_items"], 1), **st)
    assert st["coarse_fallback_items"] < 0.01 * (st["screened_items"] + st["exact_items"])
