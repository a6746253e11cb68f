"""The DUNE screening pipeline (NB_OPT_DUNE_KERNEL = 4: screen, refine, exact kernel for the flagged items) where the rest of the
suite never takes it: clouds that leave the screen's distance table, tables shrunk or refined with NB_SCREEN_TABLE_GRID, points on
the table's border and cell lines, clouds across the 512 / 1024 point kernel switches up to the shared-memory limit, points on and
inside the robot, degenerate clouds of exactly equal distances, and robots of 3, 6, 7 and 8 edges.

Two comparisons, as in test_gpu_screen.py and test_gpu_parity.py: (a) bitwise -- variant 4 against variant 2, and the table on
against off -- and (b) against the float32 oracle (oracle/dune.py) with the bars of test_dune_half_matches_oracle.  Every test
also shows that it reached the path it names, and prints what it saw as OBSERVED lines (pytest -s)."""
import contextlib
import ctypes as C
import functools
import os
import re

import numpy as np
import pytest
import torch

from gpu_helpers import make_pan, record, run_pan, to_cuda
from helpers import CONFIGS, make_inputs, robot_spec, weights_path
from neupan_b200 import _lib
from oracle import dune as od
from test_gpu_parity import TIE, TOL
from test_gpu_screen import _assert_equal

pytestmark = pytest.mark.gpu

MU_RTOL = 1e-4  # mu / lam: relative to the largest entry of the step's (M, E) / (M, 2) block (test_dune_half_matches_oracle)


# ---------------------------------------------------------------------------------------------------------------- helpers
@contextlib.contextmanager
def _grid(value):
    """NB_SCREEN_TABLE_GRID while a handle builds its table (read once, when the screening pipeline is first selected)."""
    old = os.environ.get("NB_SCREEN_TABLE_GRID")
    if value is not None:
        os.environ["NB_SCREEN_TABLE_GRID"] = value
    try:
        yield
    finally:
        if old is None:
            os.environ.pop("NB_SCREEN_TABLE_GRID", None)
        else:
            os.environ["NB_SCREEN_TABLE_GRID"] = old


def _pan(cfg, B, N, dune_kernel=4, table=None, grid=None, K=1, **kw):
    """A PAN whose native handle exists (so that the table is built under `grid`)."""
    pan = make_pan(cfg, K=K, N=N, max_envs=B, dune_kernel=dune_kernel, dune_screen_table=table, **kw)
    with _grid(grid):
        pan._ensure_handle(B, N)
    return pan


def _ptr(x):
    return None if x is None else C.c_void_p(x.data_ptr())


def _selection(pan, B):
    E = pan.dune_layer.edge_dim
    T1, M = pan.T + 1, pan.nrmp_max_num
    out = dict(mu=torch.empty(B, T1, M, E, device="cuda"), lam=torch.empty(B, T1, M, 2, device="cuda"), points=torch.empty(B, T1, M, 2, device="cuda"),
               distance=torch.empty(B, T1, M, device="cuda"), count=torch.empty(B, dtype=torch.int32, device="cuda"))
    _lib.check(_lib.load().nb_pan_read_selection(pan._handle, B, *[_ptr(out[k]) for k in ("mu", "lam", "points", "distance", "count")], None))
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def _dune(pan, inp, counts=None):
    """nb_dune_forward alone (point flow + DUNE for every step of nom_s): (selection, min_distance)."""
    B, N = inp["points"].shape[0], inp["points"].shape[-1]
    lib = pan._ensure_handle(B, N)
    t = to_cuda(dict(nom_s=inp["nom_s"], points=inp["points"], velocities=inp.get("velocities")))
    md = torch.full((B,), float("inf"), device="cuda")
    cnt = None if counts is None else torch.from_numpy(np.asarray(counts, np.int32)).cuda()
    _lib.check(lib.nb_dune_forward(pan._handle, B, N, _ptr(t["nom_s"]), _ptr(t["points"]), _ptr(t["velocities"]), _ptr(cnt), _ptr(md), None))
    torch.cuda.synchronize()
    return _selection(pan, B), md.cpu().numpy()


def _assert_same_dune(x, y):
    """(a) for two nb_dune_forward results: the same bits in every written row and the same min_distance."""
    assert np.array_equal(x[1], y[1])
    cnt = x[0]["count"]
    assert np.array_equal(cnt, y[0]["count"])
    live = np.arange(x[0]["distance"].shape[-1])[None, None, :] < cnt[:, None, None]
    for k in ("mu", "lam", "points", "distance"):
        m = live if x[0][k].ndim == 3 else live[..., None]
        assert np.array_equal(np.where(m, x[0][k], 0), np.where(m, y[0][k], 0)), k


def _pan_run(pan, inp, counts=None):
    """Full PAN forward: (S, U, D, min_distance, selection) -- the tuple test_gpu_screen._assert_equal compares."""
    if counts is None:
        S, U, D, md = run_pan(pan, inp)
    else:
        t = to_cuda(inp)
        S, U, D = pan(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"],
                      num_points=torch.from_numpy(np.asarray(counts, np.int32)).cuda())
        S, U, D, md = S.cpu().numpy(), U.cpu().numpy(), D.cpu().numpy()[:, 0], pan.min_distance.cpu().numpy()
    return (S, U, D, md, {k: v.cpu().numpy() for k, v in pan.read_selection().items()})


class Oracle:
    """oracle/dune.py for one robot and checkpoint, with the bars of test_dune_half_matches_oracle.  Only near-ties at float32
    accuracy between DIFFERENT points excuse a row (their order / membership is ambiguous); rows tied with copies of the same point
    are compared, since every copy has the same mu, lam and point."""

    def __init__(self, weights, G, h, T, dt, M):
        self.w = od.load_weights(weights)
        self.G, self.h = torch.as_tensor(np.asarray(G), dtype=torch.float32), torch.as_tensor(np.asarray(h).reshape(-1, 1), dtype=torch.float32)
        self.T, self.dt, self.M = T, dt, M
        self.worst = dict(mu=0.0, lam=0.0, dist=0.0, min_distance=0.0, rows=0, excused=0)
        self.smallest = np.inf

    @classmethod
    def of(cls, cfg):
        rb, _ = robot_spec(cfg)
        return cls(weights_path(cfg.model), rb.G, rb.h, cfg.T, cfg.dt, cfg.M)

    def check(self, inp, got, envs=None, counts=None):
        sel, md = got
        B = inp["points"].shape[0]
        for b in range(B) if envs is None else envs:
            n = inp["points"].shape[-1] if counts is None else int(counts[b])
            cnt = min(n, self.M)
            assert sel["count"][b] == cnt
            if n == 0:
                assert np.isinf(md[b])
                continue
            vel = inp.get("velocities")
            vel = None if vel is None else torch.from_numpy(np.ascontiguousarray(vel[b][:, :n]))
            p0, R, pl = od.point_flow(torch.from_numpy(inp["nom_s"][b]), torch.from_numpy(np.ascontiguousarray(inp["points"][b][:, :n])), vel,
                                      self.T, self.dt, 10 ** 9)
            mu, lam, sp, mdo, dist = od.dune_forward(self.w, self.G, self.h, p0, R, pl)
            err = abs(float(md[b]) - float(mdo))
            self.worst["min_distance"] = max(self.worst["min_distance"], err)
            assert err < 2e-5, (b, md[b], float(mdo))
            for t in range(self.T + 1):
                ds = np.sort(dist[t].numpy(), kind="stable")
                d_gpu = sel["distance"][b, t, :cnt]
                assert np.allclose(d_gpu, ds[:cnt], rtol=1e-4, atol=2e-5), (b, t, d_gpu, ds[:cnt])
                self.worst["dist"] = max(self.worst["dist"], float(np.abs(d_gpu - ds[:cnt]).max()))
                self.smallest = min(self.smallest, float(d_gpu.min()))
                pts, mu_o, lam_o = sp[t].T.numpy(), mu[t].T.numpy(), lam[t].T.numpy()
                lo = np.searchsorted(ds, ds[:cnt] - TIE, "left")
                hi = np.searchsorted(ds, ds[:cnt] + TIE, "right")
                smu, slam = max(1e-3, float(np.abs(mu_o[:cnt]).max())), max(1e-3, float(np.abs(lam_o[:cnt]).max()))
                for m in range(cnt):
                    if not (pts[lo[m]:hi[m]] == pts[m]).all():
                        self.worst["excused"] += 1
                        continue
                    self.worst["rows"] += 1
                    assert np.allclose(sel["points"][b, t, m], pts[m], atol=1e-6), (b, t, m)
                    self.worst["mu"] = max(self.worst["mu"], float(np.abs(sel["mu"][b, t, m] - mu_o[m]).max()) / smu)
                    self.worst["lam"] = max(self.worst["lam"], float(np.abs(sel["lam"][b, t, m] - lam_o[m]).max()) / slam)
        assert self.worst["mu"] < MU_RTOL and self.worst["lam"] < MU_RTOL, self.worst


def _mixed_tiles(inp, T, dt, half):
    """Screen tiles ([base, base + 32) of one item, one warp) holding points both well inside the table and well outside it: the
    points flowed and taken into each step's robot frame in float64."""
    pts, ns, vel = inp["points"].astype(np.float64), inp["nom_s"].astype(np.float64), inp.get("velocities")
    B, _, N = pts.shape
    tiles = mixed = off = 0
    for b in range(B):
        for t in range(T + 1):
            p = pts[b] if vel is None else pts[b] + t * (vel[b].astype(np.float64) * dt)
            dx, dy = p[0] - ns[b, 0, t], p[1] - ns[b, 1, t]
            c, s = np.cos(ns[b, 2, t]), np.sin(ns[b, 2, t])
            r = np.maximum(np.abs(c * dx + s * dy), np.abs(c * dy - s * dx))
            inside, outside = r < half - 1e-3, r > half + 1e-3
            for base in range(0, N, 32):
                tiles += 1
                mixed += bool(inside[base:base + 32].any() and outside[base:base + 32].any())
                off += bool(outside[base:base + 32].any())
    return mixed, tiles, off


def _scaled(inp, k):
    """The cloud stretched by k about each environment's start position."""
    s0 = inp["nom_s"][:, :2, :1]
    return dict(inp, points=np.ascontiguousarray((s0 + k * (inp["points"] - s0)).astype(np.float32)))


def _static(pts_robot, T, vel=None):
    """nom_s = (0, 0, 0) at every step: the robot frame is the world frame."""
    B = pts_robot.shape[0]
    return dict(nom_s=np.zeros((B, 3, T + 1), np.float32), points=np.ascontiguousarray(pts_robot, dtype=np.float32), velocities=vel)


# shared memory of the exact and the warpgroup screening kernels (dune_tc_smem_bytes, dune_screen_smem_bytes): operand image 31744 B,
# two 16 KB tiles, 8 B of key and 4 E B of mu per point (exact), 16 B per point (screen), 4 M candidates of 8 B, 64 B
def _tc_smem(N, E, M):
    return 31744 + 2 * 16384 + 8 * N + (N * E * 4 + 7) // 8 * 8 + 4 * M * 8 + 64


def _screen_smem(N, M):
    return 31744 + 2 * 16384 + 16 * N + 4 * M * 8 + 64


_REFUSAL = re.compile(r"N=(\d+) needs (\d+) B of shared memory \(limit (\d+)\)")


@functools.lru_cache(maxsize=None)
def _smem_limit():
    """The opt-in shared memory per block, read from the refusal of a cloud too large for the screening kernel."""
    cfg = CONFIGS["C4"]
    N = 16384
    pan = _pan(cfg, 1, N)
    z = torch.zeros(2 * N, device="cuda")
    rc = pan._ensure_handle(1, N).nb_dune_forward(pan._handle, 1, N, _ptr(torch.zeros(3 * (cfg.T + 1), device="cuda")), _ptr(z), None, None, None, None)
    msg = _lib.load().nb_last_error().decode()
    assert rc == _lib.NB_ERR_CAPACITY, (rc, msg)
    m = _REFUSAL.search(msg)
    assert m and int(m.group(1)) == N and int(m.group(2)) == _screen_smem(N, cfg.M), msg
    pan.close()
    return int(m.group(3))


def _n_max(E, M=10):
    lim = _smem_limit()
    n = (lim - _tc_smem(0, E, M)) // (8 + 4 * E)
    while _tc_smem(n + 1, E, M) <= lim:
        n += 1
    while _tc_smem(n, E, M) > lim:
        n -= 1
    return n


# ------------------------------------------------------------------------------------------------ 1. clouds that leave the table
@pytest.mark.parametrize("N", [500, 1000])
@pytest.mark.parametrize("scene", ["annulus", "obstacles"])
@pytest.mark.parametrize("cname", ["C4", "C1"])
def test_clouds_beyond_the_default_table(cname, scene, N):
    """Clouds stretched to 3..22 m: warps whose 32 points straddle the table's border run the network and keep the table's values
    for the points it covers.  N = 1000 runs the table on the 10-index-bit screen (dune_screen_mma_kernel<8>)."""
    cfg = CONFIGS[cname]
    B = 8
    inp = _scaled(make_inputs(cfg, B=B, N=N, scene=scene), 2.2)
    tab = _pan(cfg, B, N, table=1, K=3)
    a = _pan_run(tab, inp)
    info = tab.screen_table()
    assert info["bytes"] > 0
    b = _pan_run(_pan(cfg, B, N, table=0, K=3), inp)
    c = _pan_run(_pan(cfg, B, N, dune_kernel=2, K=3), inp)
    _assert_equal(a, b)
    _assert_equal(a, c)
    mixed, tiles, _ = _mixed_tiles(inp, cfg.T, cfg.dt, info["half"])
    st = tab.screen_stats()
    record("dune_edges_off_table", config=cname, scene=scene, N=N, table_half=info["half"], mixed_tiles=mixed, tiles=tiles,
           exact_items=st["exact_items"], screened_items=st["screened_items"], max_error_ratio=st["max_error_ratio"], c_mu=st["c_mu"])
    assert mixed >= 0.05 * tiles, (mixed, tiles)
    assert st["max_error_ratio"] < st["c_mu"]


# the finer grid that keeps a table on the acker and polygon checkpoints, whose 4 cm tables are dropped
FINE_GRID = "0.01,3.0"


@pytest.mark.parametrize("scene", ["annulus", "obstacles"])
@pytest.mark.parametrize("cname,grid", [("C1", "0.04,3.0"), ("C4", "0.04,3.0"), ("C2", FINE_GRID), ("C3", FINE_GRID), ("C5", FINE_GRID),
                                        ("C4", "0.04,1.5")])
def test_shrunk_table(cname, grid, scene):
    """A table of half-width 3 m: the closest points are table hits, most of the others take the network.  At 1.5 m the table
    covers little more than the robot: nearly every point, the M closest included, must take the network."""
    cfg = CONFIGS[cname]
    B = 12 if cname != "C5" else 6
    inp = make_inputs(cfg, B=B, scene=scene)
    tab = _pan(cfg, B, cfg.N, table=1, grid=grid, K=3)
    a = _pan_run(tab, inp)
    info = tab.screen_table()
    st = tab.screen_stats()
    assert abs(info["half"] - float(grid.split(",")[1])) < 0.05 and info["h"] == pytest.approx(float(grid.split(",")[0]))
    _assert_equal(a, _pan_run(_pan(cfg, B, cfg.N, table=0, K=3), inp))
    _assert_equal(a, _pan_run(_pan(cfg, B, cfg.N, dune_kernel=2, K=3), inp))
    half = float(grid.split(",")[1])
    mixed, tiles, off = _mixed_tiles(inp, cfg.T, cfg.dt, info["half"])
    record("dune_edges_shrunk_table", config=cname, scene=scene, grid=grid, table_kept=info["bytes"] > 0, table_ratio=info["max_error_ratio"],
           c_mu=st["c_mu"], mixed_tiles=mixed, tiles_with_misses=off, tiles=tiles, exact_items=st["exact_items"], max_error_ratio=st["max_error_ratio"])
    assert (info["bytes"] > 0) == (2 * info["max_error_ratio"] <= st["c_mu"])
    # kept on every checkpoint (H100, c_mu = 8e-3): diff at 4 cm with a ratio of 2.1e-3, acker and polygon at 1 cm with 3.5e-4 and 2.6e-3
    assert info["bytes"] > 0
    if half >= 3.0:
        assert mixed >= 0.05 * tiles, (mixed, tiles)
    else:
        assert off >= 0.9 * tiles, (off, tiles)


def test_points_on_the_table_border_and_cell_lines():
    """Robot frame = world frame: points exactly on x or y = +-half, one float32 step inside and outside it, on every cell line
    -half + k h and on the four corners; far points fill the rest of the cloud, so that the placed points are the M closest."""
    cfg = CONFIGS["C4"]
    T = cfg.T
    N = 160
    probe = _pan(cfg, 1, N, grid="0.04,3.0")
    info = probe.screen_table()
    assert info["bytes"] > 0
    half, h = np.float32(info["half"]), np.float32(info["h"])
    ncell = int(round(2 * float(half) / float(h)))
    edge = [half, np.nextafter(half, np.float32(0)), np.nextafter(half, np.float32(np.inf))]
    along = np.linspace(-0.9, 0.9, 19, dtype=np.float32) * half
    lines = (-half + np.arange(ncell + 1, dtype=np.float32) * h).astype(np.float32)
    sets = []
    for v in edge:  # the four borders, at the border value and one float32 step to either side
        for sgn in (1, -1):
            x = np.float32(sgn) * v
            sets.append(np.stack([np.full_like(along, x), along]))
            sets.append(np.stack([along, np.full_like(along, x)]))
    for off in (0.0, 0.37):  # every cell line, crossing the robot and off its centre
        ln = lines[np.abs(lines) >= 1.2]
        sets.append(np.stack([ln, np.full_like(ln, np.float32(off * half))]))
        sets.append(np.stack([np.full_like(ln, np.float32(off * half)), ln]))
    corners = np.array([[s * v, r * w] for s in (1, -1) for r in (1, -1) for v in edge for w in edge], np.float32).T
    sets.append(corners)
    rng = np.random.default_rng(5)
    B = len(sets)
    pts = np.zeros((B, 2, N), np.float32)
    for b, s in enumerate(sets):
        k = min(s.shape[1], N - 16)
        pick = np.sort(rng.choice(s.shape[1], k, replace=False)) if s.shape[1] > k else np.arange(k)
        ang = rng.uniform(-np.pi, np.pi, N - k)
        far = np.stack([40 * np.cos(ang), 40 * np.sin(ang)])
        allp = np.concatenate([s[:, pick], far], 1)
        pts[b] = allp[:, rng.permutation(N)]
    inp = _static(pts, T)
    tab = _pan(cfg, B, N, grid="0.04,3.0")
    on = _dune(tab, inp)
    off = _dune(_pan(cfg, B, N, table=0), inp)
    full = _dune(_pan(cfg, B, N, dune_kernel=2), inp)
    _assert_same_dune(on, off)
    _assert_same_dune(on, full)
    orc = Oracle.of(cfg)
    orc.check(inp, full)
    orc.check(inp, on)
    st = tab.screen_stats()
    record("dune_edges_table_border", half=float(half), h=float(h), envs=B, exact_items=st["exact_items"], screened_items=st["screened_items"], **orc.worst)
    assert st["screened_items"] > 0
    on_border = int((np.abs(np.abs(on[0]["points"]).max(-1) - half) <= 2e-7 * half).sum())
    record("dune_edges_table_border_rows", selected_rows_on_the_border=on_border)
    assert on_border > 0


# ---------------------------------------------------------------------------------------- 2. cloud sizes across the kernel thresholds
@pytest.mark.parametrize("N", [511, 512, 513, 1023, 1024, 1025, 2048, 4096, "max"])
@pytest.mark.parametrize("cname", ["C4", "C5"])
def test_cloud_sizes_across_kernel_switches(cname, N):
    """mma.sync screen kP = 4 / 8 up to 1024 points, the wgmma screen above; register / shared-memory keys of the exact kernel at
    512; N_max = the largest cloud the exact kernel admits."""
    cfg = CONFIGS[cname]
    N = _n_max(4, cfg.M) if N == "max" else N
    B = 4
    inp = make_inputs(cfg, B=B, N=N, scene="obstacles")
    scr, full = _pan(cfg, B, N, K=2), _pan(cfg, B, N, dune_kernel=2, K=2)
    _assert_equal(_pan_run(scr, inp), _pan_run(full, inp))
    st = scr.screen_stats()
    two = {k: (None if v is None else v[:2]) for k, v in inp.items()}
    orc = Oracle.of(cfg)
    a, b = _dune(scr, two), _dune(full, two)
    orc.check(two, a)
    orc.check(two, b)
    _assert_same_dune(a, b)
    record("dune_edges_sizes", config=cname, N=N, table_bytes=scr.screen_table()["bytes"], exact_items=st["exact_items"], screened_items=st["screened_items"], **orc.worst)
    # every item of both PAN iterations went through the screen (step 0 once), to the refine kernel or the exact kernel; above 1024
    # points the wgmma screen runs the network, whose wider intervals send almost every item of these dense clouds to the exact kernel
    assert st["exact_items"] + st["screened_items"] == B * (2 * cfg.T + 1)
    assert st["screened_items"] > 0 if N <= 1024 and cname == "C4" else st["exact_items"] > 0


def test_ragged_counts_across_switches_in_one_launch():
    cfg = CONFIGS["C4"]
    N = 2048
    counts = np.array([2048, 1025, 1024, 513, 512, 33, 32, 0], np.int32)
    B = len(counts)
    inp = make_inputs(cfg, B=B, N=N, scene="obstacles")
    scr = _pan(cfg, B, N, K=2)
    got = _pan_run(scr, inp, counts)
    _assert_equal(got, _pan_run(_pan(cfg, B, N, dune_kernel=2, K=2), inp, counts))
    assert got[4]["count"].tolist() == [10, 10, 10, 10, 10, 10, 10, 0]
    for b, n in enumerate(counts):
        one = {k: (None if v is None else np.ascontiguousarray(v[b:b + 1])) for k, v in inp.items()}
        if n:
            one["points"], one["velocities"] = np.ascontiguousarray(one["points"][..., :n]), np.ascontiguousarray(one["velocities"][..., :n])
            alone = _pan_run(_pan(cfg, 1, int(n), K=2), one)
        else:
            one["points"], one["velocities"] = one["points"][..., :1].copy(), one["velocities"][..., :1].copy()
            alone = _pan_run(_pan(cfg, 1, 1, K=2), one, [0])
        mine = tuple(x[b:b + 1] for x in got[:4]) + ({k: v[b:b + 1] for k, v in got[4].items()},)
        _assert_equal(mine, alone)
    st = scr.screen_stats()
    record("dune_edges_ragged", counts=counts.tolist(), exact_items=st["exact_items"], screened_items=st["screened_items"])


def test_one_environment_across_the_screen_switch():
    """n = 1024 through an N = 1024 launch (mma.sync screen, kP = 8, with the table) and an N = 1025 launch (wgmma screen)."""
    cfg = CONFIGS["C4"]
    inp = make_inputs(cfg, B=1, N=1024, scene="annulus")
    small = _pan(cfg, 1, 1024, K=2)
    a = _pan_run(small, inp)
    assert small.screen_table()["bytes"] > 0
    pad = dict(inp, points=np.concatenate([inp["points"], np.full((1, 2, 1), 0.5, np.float32)], -1),
               velocities=np.concatenate([inp["velocities"], np.zeros((1, 2, 1), np.float32)], -1))
    b = _pan_run(_pan(cfg, 1, 1025, K=2), pad, [1024])
    _assert_equal(a, b)


def test_shared_memory_limit_is_a_capacity_refusal():
    cfg = CONFIGS["C4"]
    lim, E, M = _smem_limit(), 4, cfg.M
    n_max = _n_max(E, M)
    n_screen = (lim - _screen_smem(0, M)) // 16
    record("dune_edges_smem", smem_limit=lim, n_max_e4=n_max, n_max_e8=_n_max(8, M), n_max_screen=n_screen)
    assert _tc_smem(n_max, E, M) <= lim < _tc_smem(n_max + 1, E, M) and n_max < n_screen
    B = 2
    inp = make_inputs(cfg, B=B, N=n_max + 1, scene="obstacles")
    at_max = dict(inp, points=np.ascontiguousarray(inp["points"][..., :n_max]), velocities=np.ascontiguousarray(inp["velocities"][..., :n_max]))
    for dk in (4, 2):
        pan = _pan(cfg, B, n_max + 1, dune_kernel=dk)
        lib = pan._ensure_handle(B, n_max + 1)
        t = to_cuda(inp)
        # nb_dune_forward: the code, and the byte count of the message against the transcription
        rc = lib.nb_dune_forward(pan._handle, B, n_max + 1, _ptr(t["nom_s"]), _ptr(t["points"]), _ptr(t["velocities"]), None, None, None)
        msg = lib.nb_last_error().decode()
        m = _REFUSAL.search(msg)
        assert rc == _lib.NB_ERR_CAPACITY and m, (rc, msg)
        assert (int(m.group(1)), int(m.group(2)), int(m.group(3))) == (n_max + 1, _tc_smem(n_max + 1, E, M), lim), msg
        # the whole forward: refused with ValueError("capacity exceeded: ..."); variant 4 has already enqueued its screen and refine
        with pytest.raises(ValueError, match="capacity exceeded: N=%d needs" % (n_max + 1)):
            run_pan(pan, inp)
        torch.cuda.synchronize()
        # the same handle afterwards, at N_max: what a fresh handle computes
        again = _pan_run(pan, at_max)
        fresh = _pan_run(_pan(cfg, B, n_max, dune_kernel=dk), at_max)
        _assert_equal(again, fresh)
        assert (pan.status.cpu().numpy() == 0).all()
    # beyond the screen's own limit the screening pipeline refuses before it launches anything
    pan = _pan(cfg, 1, n_screen + 1)
    z = torch.zeros(2 * (n_screen + 1), device="cuda")
    rc = pan._ensure_handle(1, n_screen + 1).nb_dune_forward(pan._handle, 1, n_screen + 1, _ptr(torch.zeros(3 * (cfg.T + 1), device="cuda")), _ptr(z),
                                                             None, None, None, None)
    m = _REFUSAL.search(_lib.load().nb_last_error().decode())
    assert rc == _lib.NB_ERR_CAPACITY and m and int(m.group(2)) == _screen_smem(n_screen + 1, M)


# ------------------------------------------------------------------------------------------------ 3. points on and inside the robot
def _robot_points(rb):
    """(2, k) robot-frame points: inside the polygon, exactly on its vertices and edges, 1 mm outside it."""
    V = np.asarray(rb.vertices, np.float64)  # (2, nv), counter-clockwise
    nv = V.shape[1]
    c = V.mean(1, keepdims=True)
    inside = np.concatenate([c + s * (V - c) for s in (0.0, 0.3, 0.6, 0.9)], 1)
    nxt = np.roll(V, -1, 1)
    on = np.concatenate([V] + [V + s * (nxt - V) for s in (0.25, 0.5, 0.75)], 1)
    G, h = np.asarray(rb.G, np.float64), np.asarray(rb.h, np.float64).reshape(-1)
    mid = 0.5 * (V + nxt)
    outward = []
    for j in range(nv):  # the edge's midpoint, 1 mm along the normal of the constraint it lies on
        e = int(np.argmin(np.abs(G @ mid[:, j] - h)))
        outward.append(mid[:, j] + 1e-3 * G[e] / np.linalg.norm(G[e]))
    corner = [V[:, j] + 1e-3 * (V[:, j] - c[:, 0]) / np.linalg.norm(V[:, j] - c[:, 0]) for j in range(nv)]
    return [inside.astype(np.float32), on.astype(np.float32), np.array(outward + corner, np.float32).T]


@pytest.mark.parametrize("cname", ["C4", "C5"])
def test_points_on_and_inside_the_robot(cname):
    cfg = CONFIGS[cname]
    N, T = 200, cfg.T
    rb = cfg.make_robot()
    groups = _robot_points(rb)
    base = make_inputs(cfg, B=4, N=N, scene="obstacles")
    pts = np.zeros((4, 2, N), np.float32)
    for b in range(4):  # the ordinary cloud, taken into the robot frame of its start pose
        x0, y0, th = base["nom_s"][b, :, 0].astype(np.float64)
        d = base["points"][b].astype(np.float64) - np.array([[x0], [y0]])
        c, s = np.cos(th), np.sin(th)
        pts[b] = np.stack([c * d[0] + s * d[1], -s * d[0] + c * d[1]]).astype(np.float32)
        placed = np.concatenate(groups, 1) if b == 3 else groups[b]
        pts[b, :, :placed.shape[1]] = placed
        pts[b] = pts[b][:, np.random.default_rng(b).permutation(N)]
    inp = _static(pts, T)
    orc = Oracle.of(cfg)
    runs = {}
    for dk in (4, 2):
        pan = _pan(cfg, 4, N, dune_kernel=dk)
        runs[dk] = _dune(pan, inp)
        orc.check(inp, runs[dk])
        if dk == 4:
            tab, st = pan.screen_table(), pan.screen_stats()
    off = _dune(_pan(cfg, 4, N, table=0), inp)
    _assert_same_dune(runs[4], off)
    _assert_same_dune(runs[4], runs[2])
    sel = runs[2][0]
    record("dune_edges_inside_robot", config=cname, table_kept=tab["bytes"] > 0, smallest_selected_distance=orc.smallest,
           min_distance_per_env=runs[2][1].tolist(), exact_items=st["exact_items"], **orc.worst)
    md = runs[2][1]
    assert (sel["distance"] < 0).any() and md[0] < 0 and md[3] < 0 and md[1] <= 1e-6


# ------------------------------------------------------------------------------------------------------------ 4. degenerate clouds
@pytest.mark.parametrize("N", [500, 1000])
def test_degenerate_clouds_of_equal_distances(N):
    cfg = CONFIGS["C4"]
    inp = make_inputs(cfg, B=3, N=N, scene="annulus")
    pts, vel = inp["points"].copy(), inp["velocities"].copy()
    rng = np.random.default_rng(N)
    pts[0], vel[0] = pts[0][:, :1], vel[0][:, :1]  # one point, N times
    orc = Oracle.of(cfg)
    d0 = []
    for b in (1, 2):  # the step-0 order of the distinct cloud
        _, _, _, _, dist = od.dune_forward(orc.w, orc.G, orc.h, *od.point_flow(torch.from_numpy(inp["nom_s"][b]), torch.from_numpy(inp["points"][b]),
                                                                                 torch.from_numpy(inp["velocities"][b]), cfg.T, cfg.dt, 10 ** 9))
        d0.append(np.argsort(dist[0].numpy(), kind="stable"))
    idx = rng.permutation(N)
    pts[1][:, idx[:40]], vel[1][:, idx[:40]] = pts[1][:, d0[0][:1]], vel[1][:, d0[0][:1]]  # 40 copies of the nearest point
    # two clusters: 6 copies of the nearest and 9 of the 2nd nearest point (ranks 0..5 and 6..14: across rank M = 10)
    pts[2][:, idx[:6]], vel[2][:, idx[:6]] = pts[2][:, d0[1][:1]], vel[2][:, d0[1][:1]]
    pts[2][:, idx[6:15]], vel[2][:, idx[6:15]] = pts[2][:, d0[1][1:2]], vel[2][:, d0[1][1:2]]
    inp = dict(inp, points=np.ascontiguousarray(pts), velocities=np.ascontiguousarray(vel))
    scr = _pan(cfg, 3, N)
    a = _dune(scr, inp)
    st = scr.screen_stats()
    off = _dune(_pan(cfg, 3, N, table=0), inp)
    full = _dune(_pan(cfg, 3, N, dune_kernel=2), inp)
    _assert_same_dune(a, off)
    _assert_same_dune(a, full)
    orc.check(inp, full)
    orc.check(inp, a)
    record("dune_edges_degenerate", N=N, exact_items=st["exact_items"], screened_items=st["screened_items"], **orc.worst)
    assert st["exact_items"] >= cfg.T + 2  # every item of the repeated point, and at least step 0 of the 40 copies
    assert (a[0]["distance"][1, 0] == a[0]["distance"][1, 0, 0]).all()


# ---------------------------------------------------------------------------------------------------- 5. edge counts 3, 6, 7 and 8
@functools.lru_cache(maxsize=None)
def _polygon_checkpoint(E, directory):
    from neupan_b200 import ObsPointNet

    torch.manual_seed(100 + E)
    ck = os.path.join(directory, f"model_polygon_{E}.pth")
    torch.save(ObsPointNet(2, E).state_dict(), ck)
    return ck


@pytest.mark.parametrize("E,N", [(3, 96), (3, 700), (6, 96), (6, 700), (7, 96), (7, 700), (8, 96), (8, 700), (8, "max")])
def test_edge_counts_three_and_six_to_eight(E, N, tmp_path_factory):
    from neupan_b200 import PAN, robot
    from oracle import nrmp as onr, pan as op
    from test_gpu_features import _cmp

    cfg = CONFIGS["C4"]
    N = _n_max(8, cfg.M) if N == "max" else N
    ck = _polygon_checkpoint(E, str(tmp_path_factory.getbasetemp()))
    ang = 2 * np.pi * np.arange(E) / E + 0.3
    rb = robot(cfg.T, cfg.dt, kinematics="diff", vertices=(1.2 * np.stack([np.cos(ang), np.sin(ang)], 1)).tolist(), max_speed=[8, 3], max_acce=[8, 3])
    assert rb.G.shape == (E, 2)
    B = 4
    inp = make_inputs(cfg, B=B, N=N, scene="obstacles")
    spec = onr.RobotSpec("diff", rb.G, rb.h, rb.max_speed.reshape(-1), rb.max_acce.reshape(-1), cfg.dt, None)
    w = od.load_weights(ck)
    mk = lambda: op.OraclePAN(spec, w, T=cfg.T, iter_num=1, dune_max_num=N, nrmp_max_num=cfg.M, iter_threshold=0.0, adjust=onr.Adjust(**cfg.adjust))
    ref = op.run_batch(mk, inp)
    orc = Oracle(ck, rb.G, rb.h, cfg.T, cfg.dt, cfg.M)
    new = lambda dk, table=None: PAN(cfg.T, cfg.dt, rb, iter_num=1, dune_max_num=N, nrmp_max_num=cfg.M, dune_checkpoint=ck, iter_threshold=0.0,
                                     adjust_kwargs=dict(cfg.adjust), max_envs=B, max_points=N, dune_kernel=dk, dune_screen_table=table)
    outs, worst = {}, {}
    for dk, table in ((4, 1), (4, 0), (2, None)):
        pan = new(dk, table)
        got = _pan_run(pan, inp)
        outs[(dk, table)] = got
        err = _cmp(got[:4], ref)
        bad = [b for b in range(B) if err[b] >= TOL and not _near_tie(orc, inp, b)]
        assert not bad, (dk, table, err)
        worst[f"{dk}{'' if table is None else ('t' if table else 'n')}"] = float(err.max())
        if (dk, table) == (4, 1):
            info = pan.screen_table()
            st = pan.screen_stats()
            assert st["exact_items"] + st["screened_items"] == B * (cfg.T + 1)
    _assert_equal(outs[(4, 1)], outs[(2, None)])
    _assert_equal(outs[(4, 0)], outs[(2, None)])
    record("dune_edges_polygon", E=E, N=N, table_kept=info["bytes"] > 0, table_ratio=info["max_error_ratio"], c_mu=st["c_mu"],
           exact_items=st["exact_items"], worst_rel_err=worst)


def _near_tie(orc, inp, b):
    """The environment's one PAN iteration has a near-tie at the M-th distance of some step (test_gpu_parity._excused)."""
    vel = inp.get("velocities")
    p0, R, pl = od.point_flow(torch.from_numpy(inp["nom_s"][b]), torch.from_numpy(inp["points"][b]), None if vel is None else torch.from_numpy(vel[b]),
                              orc.T, orc.dt, 10 ** 9)
    dist = od.dune_forward(orc.w, orc.G, orc.h, p0, R, pl)[4]
    for t in range(orc.T + 1):
        d = np.sort(dist[t].numpy())
        if d.shape[0] > orc.M and d[orc.M] - d[orc.M - 1] < 5 * TIE:
            return True
    return False
