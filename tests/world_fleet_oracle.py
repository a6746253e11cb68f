"""CPU restatement of the world with several robots per environment (nb_world_set_fleet), on top of tests/world_rvo_oracle.py.

Float64, the same operations in the same order as world_scan_kernel, world_fleet_step_kernel and world_rvo_kernel with K robot rows
(csrc/world_kernel.cuh, csrc/world_rvo_kernel.cuh).  ``OracleWorld`` here takes the packed scenes and behaviours of
world_rvo_oracle.OracleWorld plus the (B K, 6) robot rows of ``pack_fleet`` and K; robot k of environment b is row n = b K + k.
  * scan: a beam of robot k casts against the environment's obstacles and the edges of the other robots' bodies (the robot polygon
    at their current state, ``robot_polygon``), ids O_b + j; a robot hit reports that robot's velocity from its last step.
  * step: reactive obstacles choose first (every robot a neighbour row, after the obstacles); then Jacobi: every robot that has not
    collided integrates from the state at the start of the step, obstacles move once, and each robot's clearance is the minimum over
    the obstacles (the parents' branches) and the other robots (``clearance_robots``: both SAT orders, then the vertex-edge distances
    both ways; vectorised over the pairs of an environment in ``clearance_robot_pairs``, the same operations elementwise).
The differences from the kernels are libm's cos / sin / tan against CUDA's, in the robots' integration, bodies and velocities.
"""
import math

import numpy as np

from oracle import world as ow
import world_outline_oracle as wo
import world_rvo_oracle as wr


def clearance_robots(P, Q):
    """Robot <-> robot (lists of world vertices): the convex branch, which evaluates both SAT orders and both distance directions,
    so it is symmetric in P and Q."""
    return ow.clearance_polygon(P, Q)


def _seg_dist_v(px, py, ax, ay, bx, by):
    ex, ey, wx, wy = bx - ax, by - ay, px - ax, py - ay
    t = (wx * ex + wy * ey) / (ex * ex + ey * ey)
    t = np.where(t < 0.0, 0.0, np.where(t > 1.0, 1.0, t))
    qx, qy = wx - t * ex, wy - t * ey
    return np.sqrt(qx * qx + qy * qy)


def _separated_v(P, Q):
    """(M,) bool: an edge normal of P[m] separates P[m] and Q[m]; P, Q (M, n, 2)."""
    P1 = np.roll(P, -1, axis=1)
    nx, ny = -(P1[:, :, 1] - P[:, :, 1]), P1[:, :, 0] - P[:, :, 0]  # (M, n) one normal per edge
    pa = nx[:, :, None] * P[:, None, :, 0] + ny[:, :, None] * P[:, None, :, 1]  # (M, edge, vertex)
    pb = nx[:, :, None] * Q[:, None, :, 0] + ny[:, :, None] * Q[:, None, :, 1]
    return ((pa.max(2) < pb.min(2)) | (pb.max(2) < pa.min(2))).any(1)


def _vertex_edge_v(V, E):
    """(M,) the smallest distance from a vertex of V[m] to an edge of E[m]."""
    E1 = np.roll(E, -1, axis=1)
    d = _seg_dist_v(V[:, None, :, 0], V[:, None, :, 1], E[:, :, None, 0], E[:, :, None, 1], E1[:, :, None, 0], E1[:, :, None, 1])
    return d.reshape(len(V), -1).min(1)


def clearance_robot_pairs(P, Q):
    """clearance_robots for M pairs at once: P, Q (M, n, 2) -> (M,)."""
    sep = _separated_v(P, Q) | _separated_v(Q, P)
    d = np.minimum(_vertex_edge_v(P, Q), _vertex_edge_v(Q, P))
    return np.where(sep, np.where(d > 0.0, d, 0.0), 0.0)


def integrate(kinematics, state, action, dt, L):
    """ow.integrate plus the world-frame translation rate it used."""
    a0, a1 = float(action[0]), float(action[1])
    th = float(state[2])
    v = (a0, a1) if kinematics == "omni" else (a0 * math.cos(th), a0 * math.sin(th))
    return ow.integrate(kinematics, state, action, dt, L), v


class OracleWorld(wr.OracleWorld):
    """world_rvo_oracle.OracleWorld with K robots per environment: ``fleet`` (B K, 6) rows [start x, y, theta, goal x, y, threshold]
    (None: the env rows, K = 1)."""

    def __init__(self, cfg: dict, packed, fleet=None, K: int = 1, behaviors=None, seed: int = 0):
        super().__init__(cfg, packed, behaviors, seed)
        self.K = int(K)
        fleet = self.env[:, 4:10] if fleet is None else np.asarray(fleet, np.float64).reshape(self.B * self.K, 6)
        self.N = self.B * self.K
        self.states = fleet[:, :3].copy()
        self.fgoal = fleet[:, 3:6].copy()
        self.collided = np.zeros(self.N, np.int32)
        self.arrived = np.zeros(self.N, np.int32)
        self.fvel = np.zeros((self.N, 2))
        self.rv = np.asarray(cfg["robot_vertices"], np.float64)

    def bodies(self, b):
        return [ow.robot_polygon(self.states[b * self.K + j], self.rv) for j in range(self.K)]

    # ---- scan ----
    def scan(self, envs=None):
        """(ranges (N,R) float64, velocity (N,2,R), hit (N,R), near_tie (N,R), tangent (N,R))."""
        R, K = self.cos_a.shape[0], self.K
        envs = range(self.B) if envs is None else envs
        out = [np.zeros((self.N, R)), np.zeros((self.N, 2, R)), np.full((self.N, R), -1, np.int64), np.zeros((self.N, R), bool),
               np.zeros((self.N, R), bool)]
        for b in envs:
            o0, o1 = self.obs_begin[b], self.obs_begin[b + 1]
            nobs = o1 - o0
            circles, edges = ow.env_boundaries(self.obs, self.vert_begin, self.vertices, o0, o1)
            bodies = self.bodies(b) if K > 1 else []
            for k in range(K):
                n = b * K + k
                redges = [(*body[v], *body[(v + 1) % len(body)], nobs + j) for j, body in enumerate(bodies) if j != k for v in range(len(body))]
                E = np.concatenate([edges, np.array(redges, np.float64).reshape(-1, 5)])
                sx, sy, hc, hs = ow.sensor_ray_origin(self.states[n], self.cfg["scan_offset"])
                dx = hc * self.cos_a - hs * self.sin_a
                dy = hs * self.cos_a + hc * self.sin_a
                t, hit, tie, tan_ = ow.cast(sx, sy, dx, dy, circles, E, self.cfg["range_max"])
                out[0][n], out[2][n], out[3][n], out[4][n] = t, hit, tie, tan_
                for a in range(2):
                    ob, rb = (hit >= 0) & (hit < nobs), hit >= nobs
                    out[1][n, a][ob] = self.obs[o0 + hit[ob], 2 + a]
                    out[1][n, a][rb] = self.fvel[b * K + hit[rb] - nobs, a]
        return tuple(out)

    # ---- reactive obstacles: K robot rows ----
    def robot_rows(self, b, action):
        rows = []
        for k in range(self.K):
            n = b * self.K + k
            if self.collided[n]:
                v = (0.0, 0.0)
            else:
                a0, a1 = float(action[n][0]), float(action[n][1])
                th = float(self.states[n, 2])
                v = (a0, a1) if self.cfg["kinematics"] == "omni" else (a0 * math.cos(th), a0 * math.sin(th))
            rows.append((float(self.states[n, 0]), float(self.states[n, 1]), v[0], v[1], self.robot_r))
        return rows

    def choose_fleet(self, b, i, rows, robot_rows):
        """world_rvo_oracle.OracleWorld.choose with the K robot rows after the obstacles; the margin covers every robot's cone."""
        o = self.obs_begin[b] + i
        beh, env = self.beh[o], self.env[b]
        n = len(rows)
        allrows = rows + robot_rows
        cx, cy, vx, vy, ri = rows[i]
        gx, gy = self.goal[o]
        draws = int(self.draws[o])
        dx, dy = gx - cx, gy - cy
        dist = math.sqrt(dx * dx + dy * dy)
        margin = math.inf
        if dist < beh[9]:
            if beh[6] != 0.0:
                gx, gy = wr.draw_goal(self.seed, b, i, draws, env[:4])
                draws += 1
                dx, dy = gx - cx, gy - cy
                dist = math.sqrt(dx * dx + dy * dy)
            else:
                self.paths[o] = "parked"
                return 0.0, 0.0, (gx, gy), draws, margin
        desx = desy = 0.0
        if dist > 0.0:
            desx, desy = (beh[5] * dx) / dist, (beh[5] * dy) / dist
        cones = []
        for j in range(len(allrows)):
            if j == i:
                continue
            px, py = allrows[j][0] - cx, allrows[j][1] - cy
            D = math.sqrt(px * px + py * py)
            if D > 0.0 and D <= beh[10]:
                cones.append((j, wr.cone((cx, cy), (vx, vy), ri, allrows[j][:2], allrows[j][2:4], allrows[j][4])))
        grid, ms = beh[11], beh[12]
        lxa, lxb, hxa, hxb = vx - beh[3], -beh[1], vx + beh[3], beh[1]
        lya, lyb, hya, hyb = vy - beh[3], -beh[2], vy + beh[3], beh[2]
        lox, hix = (lxa if lxa > lxb else lxb), (hxa if hxa < hxb else hxb)
        loy, hiy = (lya if lya > lyb else lyb), (hya if hya < hyb else hyb)
        nx, ny = wr.axis_count(lox, hix, grid), wr.axis_count(loy, hiy, grid)
        k = np.arange(nx * ny)
        kx = k // ny
        ky = k - kx * ny
        ux, uy = lox + kx.astype(np.float64) * grid, loy + ky.astype(np.float64) * grid
        keep = ~(np.sqrt(ux * ux + uy * uy) < ms)
        k, ux, uy = k[keep], ux[keep], uy[keep]
        if not len(k):
            self.paths[o] = "none"
            return vx, vy, (gx, gy), draws, margin
        out = np.ones(len(k), bool)
        for j, (apex, left, right) in cones:
            wx, wy = ux - apex[0], uy - apex[1]
            c1, c2 = left[0] * wy - left[1] * wx, right[0] * wy - right[1] * wx
            out &= ~((c1 <= 0.0) & (c2 >= 0.0))
            if j >= n:
                margin = min(margin, float(np.minimum(np.abs(c1), np.abs(c2)).min()))
        ex, ey = ux - desx, uy - desy
        key = np.sqrt(ex * ex + ey * ey)
        if out.any():
            q = int(np.flatnonzero(out)[np.argmin(key[out])])
            self.paths[o] = "outside"
            return float(ux[q]), float(uy[q]), (gx, gy), draws, margin
        tmin = np.full(len(k), np.inf)
        with np.errstate(divide="ignore", invalid="ignore"):
            for j, _ in cones:
                rj = allrows[j]
                px, py, R = rj[0] - cx, rj[1] - cy, ri + rj[4]
                c = (px * px + py * py) - R * R
                if c <= 0.0:
                    tc = np.zeros(len(k))
                else:
                    wx, wy = ux - rj[2], uy - rj[3]
                    a, pw = wx * wx + wy * wy, px * wx + py * wy
                    disc = pw * pw - a * c
                    t = (pw - np.sqrt(disc)) / a
                    tc = np.where((a == 0.0) | (disc < 0.0) | ~(t > 0.0), np.inf, t)
                tmin = np.where(tc < tmin, tc, tmin)
            pen = np.where(tmin == 0.0, np.inf, beh[4] / tmin) + key
        q = int(np.argmin(pen))
        self.paths[o] = "penalty"
        if any(j >= n for j, _ in cones) and len(pen) > 1:
            p = np.sort(pen)
            margin = min(margin, float(p[1] - p[0]) if np.isfinite(p[1]) else math.inf)
        return float(ux[q]), float(uy[q]), (gx, gy), draws, margin

    def rvo(self, action, envs=None):
        margins = np.full(len(self.obs), math.inf)
        new = {}
        self.paths = {}
        for b in (range(self.B) if envs is None else envs):
            o0, o1 = self.obs_begin[b], self.obs_begin[b + 1]
            if not (self.beh[o0:o1, 0] == 1.0).any():
                continue
            rows = [(*(float(v) for v in self.obs[o, :4]), float(self.radius[o])) for o in range(o0, o1)]
            robots = self.robot_rows(b, action)
            for o in range(o0, o1):
                if self.beh[o, 0] == 1.0:
                    new[o] = self.choose_fleet(b, o - o0, rows, robots)
        for o, (vx, vy, g, d, m) in new.items():
            self.obs[o, 2], self.obs[o, 3] = vx, vy
            self.goal[o] = g
            self.draws[o] = d
            margins[o] = m
        return margins

    # ---- step ----
    def obstacle_clearance(self, body, o):
        cx, cy = self.obs[o, 0], self.obs[o, 1]
        v0, v1 = self.vert_begin[o], self.vert_begin[o + 1]
        if v1 == v0:
            return ow.clearance_circle(body, cx, cy, self.obs[o, 4])
        poly = [(cx + vx, cy + vy) for vx, vy in self.vertices[v0:v1]]
        return wo.clearance_outline(body, poly) if self.kind[o] == 1 else ow.clearance_polygon(body, poly)

    def step(self, action, rvo=True):
        """action (N,2) -> (collided, arrived, clearance (N,) float64); ``rvo=False`` skips the reactive obstacles' choice (a
        teacher-forced test runs it separately)."""
        if rvo:
            self.margins = self.rvo(action)
        cfg, K = self.cfg, self.K
        clear = np.full(self.N, np.inf)
        self.robot_clear = np.full(self.N, np.inf)  # the part of the clearance that comes from the other robots
        vel = np.zeros((self.N, 2))
        for n in range(self.N):
            if not self.collided[n]:
                self.states[n], vel[n] = integrate(cfg["kinematics"], self.states[n], action[n], cfg["step_time"], cfg.get("wheelbase"))
            gx, gy = self.states[n, 0] - self.fgoal[n, 0], self.states[n, 1] - self.fgoal[n, 1]
            if math.sqrt(gx * gx + gy * gy) < self.fgoal[n, 2]:
                self.arrived[n] = 1
        for b in range(self.B):
            o0, o1 = self.obs_begin[b], self.obs_begin[b + 1]
            for o in range(o0, o1):
                self.obs[o, :4] = ow.move_obstacle(self.obs[o], self.env[b, :4], cfg["step_time"])
            bodies = self.bodies(b)
            for k in range(K):
                for o in range(o0, o1):
                    clear[b * K + k] = min(clear[b * K + k], self.obstacle_clearance(bodies[k], o))
            if K > 1:
                ii, jj = np.nonzero(~np.eye(K, dtype=bool))
                arr = np.asarray(bodies, np.float64)
                c = clearance_robot_pairs(arr[ii], arr[jj]).reshape(K, K - 1).min(1)
                self.robot_clear[b * K:(b + 1) * K] = c
                clear[b * K:(b + 1) * K] = np.minimum(clear[b * K:(b + 1) * K], c)
        for n in range(self.N):
            if clear[n] <= 0.0:
                self.collided[n] = 1
            self.fvel[n] = (0.0, 0.0) if self.collided[n] else vel[n]
        return self.collided.copy(), self.arrived.copy(), clear
