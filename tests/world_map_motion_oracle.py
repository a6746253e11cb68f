"""Float64 restatement of obstacles in occupancy maps (nb_world_set_map_contact), TEST INFRASTRUCTURE ONLY.

``MapMotionOracleWorld`` is ``MapOracleWorld`` with the per-environment flags of ``neupan_b200.world.pack_map_contact``
(``block``).  Where a flag is 1 it adds what csrc/world_kernel.cuh and csrc/world_rvo_kernel.cuh add, with the kernels' operations
in the kernels' order:

  * ``touches``: the footprint contact test (a circle by its centre's distance to the closed cell, a convex polygon by the
    convex-convex clearance, an outline by clearance_outline with the cell as the convex side) over the occupied cells that meet the
    footprint's bounding box widened by one cell.
  * ``move``: the move rule A (the move), B (x only), C (y only), D (stay) after move_obstacle; bounces per obstacle, and the
    candidate taken counted in ``taken``.
  * ``goal_clear``: the wander goal test (footprint at the goal, and the segment to it as a two-vertex polygon at a distance > the
    circumradius from every occupied cell of its box widened by the radius and one cell); at most 16 draws per step, rejected draws
    counted in ``rejected_draws``; a bounce makes the goal count as reached at the next step.

Everything else is inherited unchanged.
"""
import math

import numpy as np

from oracle.world import _seg_dist_v, clearance_outline, clearance_robot_pairs, draw_goal, integrate, move_obstacle, robot_velocity
from world_map_oracle import MapOracleWorld, cell_polygons, map_floor

MAX_DRAWS = 16


def box_cells(table, m, x0, y0, x1, y1):
    """The occupied cells (i, j) of map m that meet [x0, x1] x [y0, y1] widened by one cell (world_map_any's range)."""
    W, H = int(table.W[m]), int(table.H[m])
    i0 = max(int(map_floor(x0, table.x0[m], table.r[m], W)) - 1, 0)
    i1 = min(int(map_floor(x1, table.x0[m], table.r[m], W)) + 1, W - 1)
    j0 = max(int(map_floor(y0, table.y0[m], table.r[m], H)) - 1, 0)
    j1 = min(int(map_floor(y1, table.y0[m], table.r[m], H)) + 1, H - 1)
    if i0 > i1 or j0 > j1:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    jj, ii = np.nonzero(table.occ[m][j0:j1 + 1, i0:i1 + 1])
    return ii + i0, jj + j0


def footprint_touches_cells(shape, cx, cy, Q):
    """(M,) bool: the footprint ``shape`` = ("circle", r) | ("convex", rel (n,2)) | ("outline", rel) centred at (cx, cy) touches
    the cells Q (M,4,2) (clearance <= 0)."""
    kind, p = shape
    if not len(Q):
        return np.zeros(0, bool)
    if kind == "circle":
        xa, ya, xb, yb = Q[:, 0, 0], Q[:, 0, 1], Q[:, 2, 0], Q[:, 2, 1]
        inside = (xa <= cx) & (cx <= xb) & (ya <= cy) & (cy <= yb)
        Q1 = np.roll(Q, -1, axis=1)
        d = _seg_dist_v(cx, cy, Q[:, :, 0], Q[:, :, 1], Q1[:, :, 0], Q1[:, :, 1]).min(1)
        return inside | (d - p <= 0.0)
    poly = np.stack([cx + p[:, 0], cy + p[:, 1]], 1)
    if kind == "convex":
        P = np.broadcast_to(poly[None], (len(Q), len(poly), 2))
        return clearance_robot_pairs(np.ascontiguousarray(P), Q) <= 0.0
    pl = [tuple(v) for v in poly]
    return np.array([clearance_outline([tuple(v) for v in q], pl) <= 0.0 for q in Q], bool)


def footprint_box(shape, cx, cy):
    kind, p = shape
    if kind == "circle":
        return cx - p, cy - p, cx + p, cy + p
    x, y = cx + p[:, 0], cy + p[:, 1]
    return x.min(), y.min(), x.max(), y.max()


def segment_near_cells(cx, cy, gx, gy, Q, rho):
    """(M,) bool: the segment (cx, cy)-(gx, gy) as a two-vertex polygon is within rho of the cells Q (clearance <= rho)."""
    if not len(Q):
        return np.zeros(0, bool)
    S = np.broadcast_to(np.array([[cx, cy], [gx, gy]], np.float64)[None], (len(Q), 2, 2))
    return clearance_robot_pairs(np.ascontiguousarray(S), Q) <= rho


class MapMotionOracleWorld(MapOracleWorld):
    def __init__(self, cfg: dict, packed, behaviors=None, seed: int = 0, *, block=None, **kw):
        super().__init__(cfg, packed, behaviors, seed, **kw)
        O = len(self.obs)
        self.block = np.zeros(self.B, np.int32) if block is None else np.asarray(block, np.int32).copy()
        self.bounces = np.zeros(O, np.int32)
        self.bounced = np.zeros(O, bool)
        self.taken = dict(B=0, C=0, D=0)
        self.rejected_draws = 0
        for b in range(self.B):
            if not self.block[b]:
                continue
            for o in range(self.obs_begin[b], self.obs_begin[b + 1]):
                if self.beh[o, 0] == 1.0 and self.beh[o, 6] != 0.0 and math.isnan(self.beh[o, 7]):
                    self.goal[o] = self.obs[o, :2]  # drawn on the first step, through the map test
                    self.draws[o] = 0

    def shape(self, o):
        v0, v1 = self.vert_begin[o], self.vert_begin[o + 1]
        if v0 == v1:
            return "circle", float(self.obs[o, 4])
        return ("outline" if self.kind[o] == 1 else "convex"), np.asarray(self.vertices[v0:v1], np.float64)

    def touches(self, b, o, cx, cy):
        m = int(self.table.env_map[b])
        sh = self.shape(o)
        i, j = box_cells(self.table, m, *footprint_box(sh, cx, cy))
        return bool(footprint_touches_cells(sh, cx, cy, cell_polygons(self.table, m, i, j)).any())

    def goal_clear(self, b, o, cx, cy, gx, gy):
        if self.touches(b, o, gx, gy):
            return False
        if gx == cx and gy == cy:
            return True
        rho = float(self.radius[o])
        m = int(self.table.env_map[b])
        i, j = box_cells(self.table, m, min(cx, gx) - rho, min(cy, gy) - rho, max(cx, gx) + rho, max(cy, gy) + rho)
        return not segment_near_cells(cx, cy, gx, gy, cell_polygons(self.table, m, i, j), rho).any()

    def choose(self, b, i, rows, robot_rows):
        o = self.obs_begin[b] + i
        beh = self.beh[o]
        if not self.block[b]:
            return super().choose(b, i, rows, robot_rows)
        cx, cy = rows[i][0], rows[i][1]
        gx, gy = self.goal[o]
        dx, dy = gx - cx, gy - cy
        if not (math.sqrt(dx * dx + dy * dy) < beh[9] or self.bounced[o]):
            return super().choose(b, i, rows, robot_rows)
        draws = int(self.draws[o])
        if beh[6] == 0.0:
            self.paths[o] = "parked"
            return 0.0, 0.0, (gx, gy), draws, math.inf
        for _ in range(MAX_DRAWS):
            g = draw_goal(self.seed, b, i, draws, self.env[b, :4])
            draws += 1
            if self.goal_clear(b, o, cx, cy, *g):
                break
            self.rejected_draws += 1
        else:
            self.paths[o] = "parked"
            return 0.0, 0.0, (cx, cy), draws, math.inf
        # the accepted goal as if it were the current one, with the threshold test off so that OracleWorld.choose does not draw again
        saved = (self.goal[o].copy(), self.draws[o], beh[9])
        self.goal[o], self.draws[o], beh[9] = g, draws, -1.0
        try:
            return super().choose(b, i, rows, robot_rows)
        finally:
            self.goal[o], self.draws[o], beh[9] = saved

    def move(self, b, o):
        """move_obstacle, then the move rule where environment b's map blocks obstacles."""
        row = self.obs[o]
        x, y, moves = float(row[0]), float(row[1]), row[2] != 0.0 or row[3] != 0.0
        cx, cy, vx, vy = move_obstacle(row, self.env[b, :4], self.cfg["step_time"])
        self.obs[o, :4] = cx, cy, vx, vy
        if not self.block[b]:
            return
        bounced = False
        if moves and self.touches(b, o, cx, cy):
            bounced = True
            self.bounces[o] += 1
            if not self.touches(b, o, cx, y):
                self.obs[o, 1], self.obs[o, 3] = y, -vy
                self.taken["B"] += 1
            elif not self.touches(b, o, x, cy):
                self.obs[o, 0], self.obs[o, 2] = x, -vx
                self.taken["C"] += 1
            else:
                self.obs[o, :4] = x, y, -vx, -vy
                self.taken["D"] += 1
        self.bounced[o] = bounced

    def obstacle_touches_map(self, o):
        """Does obstacle o touch its environment's map now (the invariant of a blocking environment's moving obstacles)?"""
        b = int(np.searchsorted(self.obs_begin, o, side="right")) - 1
        return self.touches(b, o, float(self.obs[o, 0]), float(self.obs[o, 1]))

    def step(self, action, rvo=True):
        """MapOracleWorld.step with the obstacles moved by ``move``."""
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
                self.move(b, o)
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
