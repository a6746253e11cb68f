"""The coarse bound table of the one-warp-per-item screen (dune_table_coarse_kernel, csrc/dune_table_kernel.cuh) and its two-level
selection (dune_screen_warp_kernel, csrc/dune_screen_mma_kernel.cuh), transcribed to numpy.

- The coarse bounds enclose the float32 fine bounds fl(table_bilerp - rad), fl(table_bilerp + rad) of every point of their fine cells,
  with and without fused multiply-adds in table_bilerp, at random points and on fine and coarse cell edges.
- The two-level selection (coarse keys, survivors, fine keys of the survivors) takes the same candidates in the same order as the
  one-level selection over all points, on random bound sets with ties and duplicate bounds."""
import numpy as np
import pytest

LOG = 4  # kCoarseLog
IDX = 0x1FF


def f32(x):
    return np.asarray(x, np.float64).astype(np.float32)


def round_dir(v64, dtype, down):
    """v64 rounded to dtype toward -inf (down) or +inf."""
    r = v64.astype(dtype)
    r64 = r.astype(np.float64)
    fix = (r64 > v64) if down else (r64 < v64)
    r[fix] = np.nextafter(r[fix], dtype(-np.inf) if down else dtype(np.inf))
    return r


def coarse_table(cell, rad):
    """dune_table_coarse_kernel: (cn, cn, 2) float32 {LB, UB} from fine corners (n, n, 4) and radii (n, n)."""
    n = cell.shape[0]
    cn = (n + (1 << LOG) - 1) >> LOG
    lo, hi = cell.min(-1), cell.max(-1)
    x = np.maximum(np.abs(lo), np.abs(hi)).astype(np.float64)
    m = f32(x * 2.0 ** -20 + 2.0 ** -126)
    lb = round_dir(round_dir(lo.astype(np.float64) - m, np.float32, True).astype(np.float64) - rad, np.float32, True)
    ub = round_dir(round_dir(hi.astype(np.float64) + m, np.float32, False).astype(np.float64) + rad, np.float32, False)
    pad = cn << LOG
    LB = np.full((pad, pad), np.inf, np.float32)
    UB = np.full((pad, pad), -np.inf, np.float32)
    LB[:n, :n], UB[:n, :n] = lb, ub
    LB = LB.reshape(cn, 1 << LOG, cn, 1 << LOG).min(axis=(1, 3))
    UB = UB.reshape(cn, 1 << LOG, cn, 1 << LOG).max(axis=(1, 3))
    hl = round_dir(LB.astype(np.float64), np.float16, True).astype(np.float32)
    hu = round_dir(UB.astype(np.float64), np.float16, False).astype(np.float32)
    hl[hl == 0] = -0.0
    hu[hu == 0] = 0.0
    return np.stack([hl, hu], -1)


def fma32(a, b, c):
    return f32(a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64))


def bilerp(c, a, b, fused):
    """table_bilerp in float32 (dune_common.cuh), with or without contraction of its three multiply-adds."""
    mad = fma32 if fused else (lambda p, q, r: (p * q).astype(np.float32) + r)
    d0 = mad(a, c[..., 1] - c[..., 0], c[..., 0])
    d1 = mad(a, c[..., 3] - c[..., 2], c[..., 2])
    return mad(b, d1 - d0, d0)


def synthetic_table(n, rng):
    """Corners of very different magnitudes and signs, flat cells (all four corners equal) and radii down to the table's floor."""
    base = rng.standard_normal((n + 1, n + 1)) * 10.0 ** rng.integers(-3, 3, (n + 1, n + 1))
    corners = np.stack([base[:-1, :-1], base[:-1, 1:], base[1:, :-1], base[1:, 1:]], -1).astype(np.float32)
    flat = rng.random((n, n)) < 0.2
    corners[flat] = corners[flat][:, :1]
    rad = f32(10.0 ** rng.uniform(-4, -1, (n, n)))
    return corners, rad


@pytest.mark.parametrize("n", [100, 820])
@pytest.mark.parametrize("fused", [True, False])
def test_coarse_bounds_enclose_the_fine_bounds(n, fused):
    rng = np.random.default_rng(n + fused)
    cell, rad = synthetic_table(n, rng)
    co = coarse_table(cell, rad)
    # points: random cells at random positions, and every cell at its edges (a, b in {0, largest float below 1})
    k = 400_000
    iy, ix = rng.integers(0, n, k), rng.integers(0, n, k)
    a, b = rng.random(k, dtype=np.float32), rng.random(k, dtype=np.float32)
    edge = np.array([0.0, np.nextafter(np.float32(1), np.float32(0))], np.float32)
    gy, gx, ea, eb = np.meshgrid(np.arange(n), np.arange(n), edge, edge, indexing="ij")
    iy, ix = np.concatenate([iy, gy.ravel()]), np.concatenate([ix, gx.ravel()])
    a, b = np.concatenate([a, ea.ravel()]), np.concatenate([b, eb.ravel()])
    d = bilerp(cell[iy, ix], a, b, fused)
    r = rad[iy, ix]
    lb_f, ub_f = d - r, d + r
    c = co[iy >> LOG, ix >> LOG]
    assert np.all(c[:, 0] <= lb_f) and np.all(c[:, 1] >= ub_f)


def test_coarse_table_covers_the_last_partial_row_and_column():
    rng = np.random.default_rng(5)
    cell, rad = synthetic_table(820, rng)
    co = coarse_table(cell, rad)
    assert co.shape[:2] == (52, 52)  # 820 = 51 x 16 + 4
    last = slice(51 << LOG, 820)
    lo = (cell[last, last].min(-1) - rad[last, last]).min()
    hi = (cell[last, last].max(-1) + rad[last, last]).max()
    assert lo - 0.01 * abs(lo) - 1e-3 <= co[51, 51, 0] <= lo and hi <= co[51, 51, 1] <= hi + 0.01 * abs(hi) + 1e-3


def orderable(x):
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    o = np.where(u & 0x80000000, ~u & 0xFFFFFFFF, u | 0x80000000)
    return np.where(np.isnan(x), 0xFFFFFFFF, o).astype(np.uint64)


def unique_key(k, i):
    return (((np.minimum(k, 0xFFFFF000) + IDX + 1) & ~np.uint64(IDX)) | i.astype(np.uint64)).astype(np.uint64)


def lane_order(n):
    """The kernel's order of points: tile j = i // 32, then lane 4 g + tq of the point 8 tq + g it owns."""
    i = np.arange(n)
    own = i % 32
    return np.lexsort(((own % 8) * 4 + own // 8, i // 32))


def select(lb, ub, M, order, mask=None):
    """Candidates of the one-level selection over the points in mask, in the kernel's order."""
    i = np.arange(lb.size)
    mask = np.ones(lb.size, bool) if mask is None else mask
    key = np.where(mask, unique_key(orderable(ub), i), 0xFFFFFFFF)
    tau = np.sort(key)[M - 1]
    take = mask & (orderable(lb) <= tau)
    return [p for p in order if take[p]]


@pytest.mark.parametrize("M", [1, 10, 32])
@pytest.mark.parametrize("n", [33, 100, 500, 512])
def test_two_level_selection_equals_one_level_selection(n, M):
    rng = np.random.default_rng(1000 * n + M)
    order = lane_order(n)
    for trial in range(200):
        # distances quantized to few values (ties) and radii from a small set (duplicate bounds)
        d = f32(np.round(rng.uniform(-0.5, 6.0, n) * rng.choice([4, 16, 256])) / 16)
        r = f32(rng.choice([1e-4, 0.01, 0.05, 0.2], n))
        lb_f, ub_f = (d - r).astype(np.float32), (d + r).astype(np.float32)
        # coarse bounds: points share a coarse cell's bounds (the min / max over their group), widened a little
        g = rng.integers(0, max(2, n // rng.choice([2, 8, 40])), n)
        glb = np.full(g.max() + 1, np.inf, np.float32)
        gub = np.full(g.max() + 1, -np.inf, np.float32)
        np.minimum.at(glb, g, lb_f)
        np.maximum.at(gub, g, ub_f)
        lb_c = f32(glb[g] - rng.choice([0.0, 1e-3, 0.3], n))
        ub_c = f32(gub[g] + rng.choice([0.0, 1e-3, 0.3], n))
        assert np.all(lb_c <= lb_f) and np.all(ub_c >= ub_f)
        one = select(lb_f, ub_f, M, order)
        i = np.arange(n)
        tau_c = np.sort(unique_key(orderable(ub_c), i))[M - 1]
        surv = orderable(lb_c) <= tau_c
        two = select(lb_f, ub_f, M, order, mask=surv)
        assert two == one, trial
