"""Float64 restatement of occupancy maps in the batched world (nb_world_set_maps), TEST INFRASTRUCTURE ONLY.

``MapOracleWorld`` is ``MixedOracleWorld`` (so ``OracleWorld`` when there are no robot types) with the maps of
``neupan_b200.world.pack_maps``: ``maps=(maps, bits, env_map)`` and the handle's ``window``.  It adds what csrc/world_kernel.cuh adds,
with the kernels' operations in the kernels' order:

  * ``map_cast``: the grid walk of world_map_cast, vectorised over beams (every beam's t from its cell index, never accumulated;
    the corner rule; the sensor's cell by floor and one correction step), run after the shape and robot tests with
    lim = min(best, range_max); a crossing before lim is hit index O_b + K with velocity 0.
  * ``map_clearance``: world_map_clearance, the convex-convex clearance (clearance_robot_pairs, whose SAT and vertex-edge distances
    are the kernels') to every occupied cell of the window range, each cell the CCW square of its four grid lines; then
    min(window, that).

Everything else (obstacles, robots, reactive obstacles, robot types) is inherited unchanged.
"""
import math

import numpy as np

from oracle.world import clearance_robot_pairs, integrate, move_obstacle, robot_velocity, sensor_ray_origin
from world_mixed_oracle import MixedOracleWorld


def map_line(lo, r, k):
    """Grid line k: lo + k r, each operation rounded (world_map_line); k an int array."""
    return lo + np.asarray(k).astype(np.float64) * r


def map_floor(s, lo, r, n):
    """floor((s - lo) / r) clamped to -1..n (world_map_floor)."""
    f = np.floor((s - lo) / r)
    return np.where(f < -1.0, -1.0, np.where(f > n, n, f)).astype(np.int64)


def map_cell(s, lo, r, n):
    """world_map_cell: map_floor corrected by one step so that line(i) <= s < line(i + 1)."""
    i = map_floor(s, lo, r, n)
    dec = (i > -1) & (s < map_line(lo, r, i))
    inc = ~dec & (i < n) & (s >= map_line(lo, r, i + 1))
    return i - dec + inc


def map_next(s, d, lo, r, i, n):
    """world_map_next: (t, ni) of the next grid line on this axis; t = inf where d == 0."""
    k = np.where(d > 0.0, np.where(i < 0, 0, i + 1), np.where(i >= n, n, i))
    ni = np.where(d > 0.0, k, k - 1)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.where(d != 0.0, (map_line(lo, r, k) - s) / np.where(d != 0.0, d, 1.0), np.inf)
    return t, ni


class MapTable:
    """The maps of pack_maps, unpacked: per map (W, H, x0, y0, r) and its cells as one flat bool array (row j = y index j)."""

    def __init__(self, maps, bits, env_map):
        self.env_map = np.asarray(env_map, np.int64)
        P = int(self.env_map.max()) + 1 if len(self.env_map) and self.env_map.max() >= 0 else 0
        bits = np.asarray(bits, np.uint32)
        self.W, self.H, self.x0, self.y0, self.r, self.coff, self.occ = [], [], [], [], [], [], []
        woff, coff = 0, 0
        for p in range(P):
            m = maps[p]
            W, H = int(m.width), int(m.height)
            words = (W + 31) // 32
            chunk = bits[woff:woff + H * words].astype("<u4").view(np.uint8).reshape(H, 4 * words)
            occ = np.unpackbits(chunk, axis=1, bitorder="little")[:, :W].astype(bool)
            self.occ.append(occ)
            self.W.append(W); self.H.append(H)
            self.x0.append(float(m.origin[0])); self.y0.append(float(m.origin[1])); self.r.append(float(m.resolution))
            self.coff.append(coff)
            woff += H * words
            coff += H * W
        self.flat = np.concatenate([o.reshape(-1) for o in self.occ]) if self.occ else np.zeros(1, bool)
        for name in ("W", "H", "coff"):
            setattr(self, name, np.asarray(getattr(self, name), np.int64))
        for name in ("x0", "y0", "r"):
            setattr(self, name, np.asarray(getattr(self, name), np.float64))

    def occupied(self, m, i, j):
        W, H = self.W[m], self.H[m]
        inside = (i >= 0) & (i < W) & (j >= 0) & (j < H)
        return inside & self.flat[np.where(inside, self.coff[m] + j * W + i, 0)]


def map_cast(table, m, sx, sy, dx, dy, lim):
    """world_map_cast for beams (arrays; m the map of each beam): t of the first state change in (0, lim), inf where none."""
    x0, y0, r, W, H = table.x0[m], table.y0[m], table.r[m], table.W[m], table.H[m]
    i, j = map_cell(sx, x0, r, W), map_cell(sy, y0, r, H)
    cur = table.occupied(m, i, j)
    tx, ni = map_next(sx, dx, x0, r, i, W)
    ty, nj = map_next(sy, dy, y0, r, j, H)
    out = np.full(len(sx), np.inf)
    act = np.arange(len(sx))
    while len(act):
        out_x = ((i < 0) & ~(dx > 0.0)) | ((i >= W) & ~(dx < 0.0)) | ((j < 0) & ~(dy > 0.0)) | ((j >= H) & ~(dy < 0.0))
        t = np.minimum(tx, ty)
        go = ~out_x & (t < lim)
        xs, ys = tx < ty, ty < tx
        cs = ~xs & ~ys
        a, c, s = table.occupied(m, ni, j), table.occupied(m, i, nj), table.occupied(m, ni, nj)
        new = np.where(xs, a, np.where(ys, c, s))
        changed = np.where(cs, (a != cur) | (c != cur) | (s != cur), new != cur)
        hit = go & changed & (t > 0.0)
        out[act[hit]] = t[hit]
        keep = go & ~hit
        i2, j2 = np.where(ys, i, ni), np.where(xs, j, nj)
        tx2, ni2 = map_next(sx, dx, x0, r, i2, W)
        ty2, nj2 = map_next(sy, dy, y0, r, j2, H)
        tx, ni = np.where(ys, tx, tx2), np.where(ys, ni, ni2)
        ty, nj = np.where(xs, ty, ty2), np.where(xs, nj, nj2)
        i, j, cur = i2, j2, new
        sel = np.flatnonzero(keep)
        act = act[sel]
        (sx, sy, dx, dy, lim, m, x0, y0, r, W, H, i, j, cur, tx, ty, ni, nj) = (
            v[sel] for v in (sx, sy, dx, dy, lim, m, x0, y0, r, W, H, i, j, cur, tx, ty, ni, nj))
    return out


def window_cells(table, m, body, window):
    """The occupied cells (i, j) of map m in world_map_clearance's range for the body (list of world vertices)."""
    xs, ys = [v[0] for v in body], [v[1] for v in body]
    xmin, xmax, ymin, ymax = min(xs), max(xs), min(ys), max(ys)
    W, H = int(table.W[m]), int(table.H[m])
    i0 = max(int(map_floor(xmin - window, table.x0[m], table.r[m], W)) - 1, 0)
    i1 = min(int(map_floor(xmax + window, table.x0[m], table.r[m], W)) + 1, W - 1)
    j0 = max(int(map_floor(ymin - window, table.y0[m], table.r[m], H)) - 1, 0)
    j1 = min(int(map_floor(ymax + window, table.y0[m], table.r[m], H)) + 1, H - 1)
    if i0 > i1 or j0 > j1:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    jj, ii = np.nonzero(table.occ[m][j0:j1 + 1, i0:i1 + 1])
    return ii + i0, jj + j0


def cell_polygons(table, m, i, j):
    """(M, 4, 2) the CCW squares of cells (i, j) of map m: (xa, ya), (xb, ya), (xb, yb), (xa, yb)."""
    xa, xb = map_line(table.x0[m], table.r[m], i), map_line(table.x0[m], table.r[m], i + 1)
    ya, yb = map_line(table.y0[m], table.r[m], j), map_line(table.y0[m], table.r[m], j + 1)
    return np.stack([np.stack([xa, ya], 1), np.stack([xb, ya], 1), np.stack([xb, yb], 1), np.stack([xa, yb], 1)], 1)


def map_clearance(table, m, body, window):
    """world_map_clearance then min(window, .): the body's clearance to map m, exact up to window."""
    i, j = window_cells(table, m, body, window)
    if not len(i):
        return float(window)
    Q = cell_polygons(table, m, i, j)
    d = math.inf
    for c0 in range(0, len(Q), 65536):
        q = Q[c0:c0 + 65536]
        P = np.broadcast_to(np.asarray(body, np.float64)[None], (len(q), len(body), 2))
        d = min(d, float(clearance_robot_pairs(np.ascontiguousarray(P), q).min()))
    return min(float(window), d)


class MapOracleWorld(MixedOracleWorld):
    def __init__(self, cfg: dict, packed, behaviors=None, seed: int = 0, *, fleet=None, K: int = 1, types=(), robot_type=None, maps=None,
                 window: float = 1.0):
        super().__init__(cfg, packed, behaviors, seed, fleet=fleet, K=K, types=types, robot_type=robot_type)
        self.table = MapTable(*maps) if maps is not None else MapTable([], np.zeros(1, np.uint32), np.full(self.B, -1))
        self.window = float(window)
        self.map_clear = np.full(self.N, np.inf)  # the map term of the last step's clearance

    def scan(self, envs=None):
        """OracleWorld's scan, then each environment's map with lim = the range found so far (index O_b + K, velocity 0)."""
        out = super().scan(envs)
        R, K = self.cos_a.shape[0], self.K
        envs = range(self.B) if envs is None else envs
        rows, mids, sxs, sys_, dxs, dys = [], [], [], [], [], []
        for b in envs:
            mi = int(self.table.env_map[b])
            if mi < 0:
                continue
            for k in range(K):
                n = b * K + k
                sx, sy, hc, hs = sensor_ray_origin(self.states[n], self.cfg["scan_offset"])
                rows.append(np.full(R, n)); mids.append(np.full(R, mi))
                sxs.append(np.full(R, sx)); sys_.append(np.full(R, sy))
                dxs.append(hc * self.cos_a - hs * self.sin_a); dys.append(hs * self.cos_a + hc * self.sin_a)
        if not rows:
            return out
        n, m = np.concatenate(rows), np.concatenate(mids)
        beam = np.tile(np.arange(R), len(rows))
        lim = out[0][n, beam]
        t = map_cast(self.table, m, np.concatenate(sxs), np.concatenate(sys_), np.concatenate(dxs), np.concatenate(dys), lim)
        hit = t < lim
        n, beam = n[hit], beam[hit]
        out[0][n, beam] = t[hit]
        out[2][n, beam] = np.diff(self.obs_begin)[n // K] + K
        out[1][n, 0, beam] = 0.0
        out[1][n, 1, beam] = 0.0
        out[3][n, beam] = False  # the map is not part of OracleWorld's near-tie diagnostics
        return out

    def map_clearances(self, bodies):
        """(N,) min(window, the clearance to the environment's map) of every robot (inf without a map), bodies a list of N."""
        out = np.full(self.N, np.inf)
        for n in range(self.N):
            mi = int(self.table.env_map[n // self.K])
            if mi >= 0:
                out[n] = map_clearance(self.table, mi, bodies[n], self.window)
        return out

    def step(self, action, rvo=True):
        """MixedOracleWorld.step with the map term: action (N,2) -> (collided, arrived, clearance (N,) float64)."""
        if rvo:
            self.margins = self.rvo(action)
        cfg, K = self.cfg, self.K
        clear = np.full(self.N, np.inf)
        self.robot_clear = np.full(self.N, np.inf)
        vel = np.zeros((self.N, 2))
        for n in range(self.N):
            if not self.collided[n]:
                kin, L, _, _ = self.type_of(n)
                vel[n] = robot_velocity(kin, action[n], float(self.states[n, 2]))
                self.states[n] = integrate(kin, self.states[n], action[n], cfg["step_time"], L)
            gx, gy = self.states[n, 0] - self.fgoal[n, 0], self.states[n, 1] - self.fgoal[n, 1]
            if math.sqrt(gx * gx + gy * gy) < self.fgoal[n, 2]:
                self.arrived[n] = 1
        every = []
        for b in range(self.B):
            o0, o1 = self.obs_begin[b], self.obs_begin[b + 1]
            for o in range(o0, o1):
                self.obs[o, :4] = move_obstacle(self.obs[o], self.env[b, :4], cfg["step_time"])
            bodies = self.bodies(b)
            every += bodies
            for k in range(K):
                for o in range(o0, o1):
                    clear[b * K + k] = min(clear[b * K + k], self.obstacle_clearance(bodies[k], o))
        if K > 1:
            self.robot_clear = self.robot_clearances(every)
            clear = np.minimum(clear, self.robot_clear)
        self.map_clear = self.map_clearances(every)
        clear = np.minimum(clear, self.map_clear)
        for n in range(self.N):
            if clear[n] <= 0.0:
                self.collided[n] = 1
            self.fvel[n] = (0.0, 0.0) if self.collided[n] else vel[n]
        return self.collided.copy(), self.arrived.copy(), clear
