"""CPU check of the screen's distance table (csrc/dune_table_kernel.cuh, table_lookup / table_bilerp in csrc/dune_common.cuh),
transcribed to numpy: cells from a grid sampled kTableSub times finer, the cell's radius from the fine samples, the lookup's bilinear
interpolation.  With the network of every shipped checkpoint, the radius must bound the interpolation error at points the build never
sampled, and the table's error ratio must stay below the smallest screening bound a handle uses (c_mu >= 0.008) wherever a scene can
place a point."""
import numpy as np
import pytest
import torch

from helpers import CONFIGS, weights_path
from oracle import dune as od

SUB, SAFETY, FLOOR = 4, 4.0, 1e-4  # kTableSub, kTableSafety, kTableFloor
H = 0.04                           # default cell side (NB_SCREEN_TABLE_GRID)
C_MU_MIN = 0.008                   # the smallest c_mu calibrate_screen() sets


def bilerp(c, a, b):
    d0 = c[..., 0] + a * (c[..., 1] - c[..., 0])
    d1 = c[..., 2] + a * (c[..., 3] - c[..., 2])
    return d0 + b * (d1 - d0)


def build(dist, x0, y0, n, h):
    """cells (n, n, 4) and radii (n, n) of the table whose cell (0, 0) starts at (x0, y0)"""
    m = SUB * n + 1
    u = np.arange(m) * (h / SUB)
    X, Y = np.meshgrid(x0 + u, y0 + u, indexing="xy")  # f[v, u]
    f = dist(np.stack([X.ravel(), Y.ravel()], 1)).reshape(m, m)
    c = np.stack([f[:-1:SUB, :-1:SUB], f[:-1:SUB, SUB::SUB], f[SUB::SUB, :-1:SUB], f[SUB::SUB, SUB::SUB]], -1)
    fp = np.pad(f, 1, mode="edge")  # at the grid border the missing neighbour is the sample itself (as in the kernel)
    d2 = np.maximum(np.abs(fp[1:-1, 2:] - 2 * f + fp[1:-1, :-2]), np.abs(fp[2:, 1:-1] - 2 * f + fp[:-2, 1:-1]))
    err, cd2 = np.zeros((n, n)), np.zeros((n, n))
    for t in range(SUB + 1):
        for s in range(SUB + 1):
            err = np.maximum(err, np.abs(bilerp(c, s / SUB, t / SUB) - f[t::SUB, s::SUB][:n, :n]))
            cd2 = np.maximum(cd2, d2[t::SUB, s::SUB][:n, :n])
    return c, SAFETY * (err + cd2) + FLOOR


def lookup(c, rad, x0, y0, h, P):
    fx, fy = (P[:, 0] - x0) / h, (P[:, 1] - y0) / h
    ix, iy = np.floor(fx).astype(int), np.floor(fy).astype(int)
    return bilerp(c[iy, ix], fx - ix, fy - iy), rad[iy, ix]


def test_bilerp_reproduces_the_corners_and_linear_fields():
    c = np.array([1.0, 2.0, 5.0, 7.0])
    assert [bilerp(c, a, b) for a, b in ((0, 0), (1, 0), (0, 1), (1, 1))] == [1.0, 2.0, 5.0, 7.0]
    lin = lambda P: 0.3 * P[:, 0] - 1.2 * P[:, 1] + 0.5  # bilinear interpolation is exact on it: every radius is the floor
    cells, rad = build(lin, -1.0, -1.0, 8, 0.25)
    assert np.allclose(rad[1:-1, 1:-1], FLOOR)  # the border cells see the grid edge as a kink
    P = np.random.default_rng(0).uniform(-1, 1, (1000, 2))
    d, _ = lookup(cells, rad, -1.0, -1.0, 0.25, P)
    assert np.allclose(d, lin(P), atol=1e-12)


@pytest.mark.parametrize("model", sorted({cfg.model for cfg in CONFIGS.values()}))
def test_table_radius_bounds_the_interpolation_error(model):
    cfg = next(c for c in CONFIGS.values() if c.model == model)
    rb = cfg.make_robot()
    G, hh = np.asarray(rb.G, np.float64), np.asarray(rb.h, np.float64).reshape(-1)
    w = od.load_weights(weights_path(model))

    def dist(P):
        with torch.no_grad():
            mu = od.obs_point_net(w, torch.from_numpy(P.astype(np.float32))).double().numpy()
        return np.einsum("ne,ne->n", mu, P @ G.T - hh)

    # the 8 m x 8 m window around the robot: the polygon's corners, where the network's ReLU kinks make the largest errors
    half, n = 4.0, int(round(8.0 / H))
    cells, rad = build(dist, -half, -half, n, H)
    P = np.random.default_rng(1).uniform(-half, half - 1e-6, (100000, 2))
    d, r = lookup(cells, rad, -half, -half, H, P)
    err = np.abs(d - dist(P))
    sa = np.abs(P @ G.T - hh).sum(1)
    assert np.all(err <= 0.5 * r), (err / r).max()  # the refine kernel's run-time check would never fire
    # the statistic nb_pan_read_screen_stats compares with c_mu, at the points a scene can hold (outside the polygon inflated by 0.2 m)
    outside = np.any(P @ G.T - hh > 0.2 * np.linalg.norm(G, axis=1), axis=1)
    assert (err / sa)[outside].max() < C_MU_MIN, (err / sa)[outside].max()
