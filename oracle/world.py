"""CPU restatement of the batched 2-D world (TEST INFRASTRUCTURE ONLY, like the rest of oracle/).

Float64, the same operations in the same order as csrc/world_kernel.cuh (which rounds every product and sum separately, no FMA),
so that the kernels agree with it to the last bit wherever their inputs agree; the only differences come from CUDA's sin / cos /
tan vs libm.  Inputs are the packed arrays of ``neupan_b200.world.pack_scenes`` and a config dict:

    kinematics ("diff" | "acker" | "omni"), step_time, wheelbase, angle_min, angle_max, range_max, number (R),
    scan_offset (3,), robot_vertices (n, 2) in the robot frame.

Geometry:
  * ray / circle: |s + t d - c|^2 = r^2 with |d| = 1:  t = -b -+ sqrt(b^2 - c'),  b = (s - c).d,  c' = |s - c|^2 - r^2
  * ray / segment a->b:  s + t d = a + u e,  e = b - a,  w = a - s:  t = (w x e) / (d x e),  u = (w x d) / (d x e),  0 <= u <= 1
  * the range is the smallest t > 0 over all boundaries (equal t: the lower obstacle index); none below range_max: range_max, hit -1
  * clearance robot polygon <-> circle: distance from the centre to the polygon (0 inside) - r;  <-> convex polygon: 0 unless an
    edge normal of either polygon separates them (SAT), else the smallest vertex-edge distance;  clamped at 0
"""
import math

import numpy as np

KIN = {"diff": 0, "acker": 1, "omni": 2}


def beam_table(angle_min, angle_max, R):
    """cos / sin of numpy.linspace(angle_min, angle_max, R), with libm (math.cos / math.sin)."""
    a = np.linspace(angle_min, angle_max, R)
    return np.array([math.cos(v) for v in a]), np.array([math.sin(v) for v in a])


def sensor_ray_origin(state, scan_offset):
    """Sensor position and (cos, sin) of its heading for the robot state (x, y, theta)."""
    x, y, th = (float(v) for v in state)
    cs, sn = math.cos(th), math.sin(th)
    sx = x + (cs * scan_offset[0] - sn * scan_offset[1])
    sy = y + (sn * scan_offset[0] + cs * scan_offset[1])
    h = th + scan_offset[2]
    return sx, sy, math.cos(h), math.sin(h)


def env_boundaries(obs, vert_begin, vertices, o0, o1):
    """The environment's circles (cx, cy, r, local index) and polygon edges (ax, ay, bx, by, local index) in world coordinates."""
    circles, edges = [], []
    for o in range(o0, o1):
        cx, cy = obs[o, 0], obs[o, 1]
        v0, nv = vert_begin[o], vert_begin[o + 1] - vert_begin[o]
        if nv == 0:
            circles.append((cx, cy, obs[o, 4], o - o0))
        for k in range(nv):
            k1 = (k + 1) % nv
            edges.append((cx + vertices[v0 + k, 0], cy + vertices[v0 + k, 1], cx + vertices[v0 + k1, 0], cy + vertices[v0 + k1, 1], o - o0))
    return np.array(circles, np.float64).reshape(-1, 4), np.array(edges, np.float64).reshape(-1, 5)


def cast(sx, sy, dx, dy, circles, edges, range_max):
    """Ray casts from (sx, sy) along the unit directions (dx, dy) (R,).  Returns (t (R,) float64, hit (R,) int64, and the
    diagnostics near_tie (R,) bool = two crossings within 1e-9 m of the first one, tangent (R,) bool = a circle whose
    |discriminant| is below 1e-12 of b^2)."""
    R = dx.shape[0]
    dx, dy = dx[:, None], dy[:, None]
    with np.errstate(invalid="ignore", divide="ignore"):
        cx, cy, r, cid = circles[:, 0], circles[:, 1], circles[:, 2], circles[:, 3]
        fx, fy = sx - cx, sy - cy
        bq = fx * dx + fy * dy
        cq = (fx * fx + fy * fy) - r * r
        disc = bq * bq - cq
        sq = np.sqrt(np.where(disc >= 0.0, disc, 0.0))
        t1, t2 = -bq - sq, -bq + sq
        tc = np.where(t1 > 0.0, t1, t2)
        tc = np.where((disc >= 0.0) & (tc > 0.0), tc, np.inf)
        tangent = (np.abs(disc) < 1e-12 * np.maximum(bq * bq, 1e-300)).any(1)
        ax, ay, bx, by, eid = (edges[:, i] for i in range(5))
        ex, ey = bx - ax, by - ay
        den = dx * ey - dy * ex
        wx, wy = ax - sx, ay - sy
        te = (wx * ey - wy * ex) / den
        u = (wx * dy - wy * dx) / den
        te = np.where((den != 0.0) & (u >= 0.0) & (u <= 1.0) & (te > 0.0), te, np.inf)
    t = np.concatenate([tc, te], 1)
    ids = np.concatenate([np.broadcast_to(cid, tc.shape), np.broadcast_to(eid, te.shape)], 1)
    best = t.min(1) if t.shape[1] else np.full(R, np.inf)
    hit = np.where(t == best[:, None], ids, np.inf).min(1) if t.shape[1] else np.full(R, np.inf)
    # another crossing (of a different obstacle, or the same obstacle's boundary elsewhere) within 1e-9 m of the first one
    with np.errstate(invalid="ignore"):
        close = np.isfinite(t) & (np.abs(t - best[:, None]) <= 1e-9)
    near_tie = (close & (ids != hit[:, None])).any(1) if t.shape[1] else np.zeros(R, bool)
    miss = ~(best < range_max)
    best = np.where(miss, range_max, best)
    hit = np.where(miss, -1, hit).astype(np.int64)
    return best, hit, near_tie & ~miss, tangent


def seg_dist(px, py, ax, ay, bx, by):
    """Distance from p to the segment a-b."""
    ex, ey, wx, wy = bx - ax, by - ay, px - ax, py - ay
    t = (wx * ex + wy * ey) / (ex * ex + ey * ey)
    t = 0.0 if t < 0.0 else (1.0 if t > 1.0 else t)
    qx, qy = wx - t * ex, wy - t * ey
    return math.sqrt(qx * qx + qy * qy)


def _separated(P, Q):
    """Does an edge normal of polygon P separate P and Q (lists of (x, y))?"""
    n = len(P)
    for k in range(n):
        k1 = (k + 1) % n
        nx, ny = -(P[k1][1] - P[k][1]), P[k1][0] - P[k][0]
        pa = [nx * x + ny * y for x, y in P]
        pb = [nx * x + ny * y for x, y in Q]
        if max(pa) < min(pb) or max(pb) < min(pa):
            return True
    return False


def clearance_circle(robot, cx, cy, r):
    """Robot polygon (list of world vertices) <-> circle."""
    pos = neg = False
    d = math.inf
    n = len(robot)
    for k in range(n):
        (ax, ay), (bx, by) = robot[k], robot[(k + 1) % n]
        cr = (bx - ax) * (cy - ay) - (by - ay) * (cx - ax)
        pos, neg = pos or cr > 0.0, neg or cr < 0.0
        d = min(d, seg_dist(cx, cy, ax, ay, bx, by))
    c = d - r if (pos and neg) else 0.0  # the centre inside the robot: overlap
    return c if c > 0.0 else 0.0


def clearance_polygon(robot, poly):
    """Robot polygon <-> convex polygon (lists of world vertices)."""
    if not (_separated(robot, poly) or _separated(poly, robot)):
        return 0.0
    d = math.inf
    for A, B in ((poly, robot), (robot, poly)):  # vertices of B against the edges of A
        for k in range(len(A)):
            (ax, ay), (bx, by) = A[k], A[(k + 1) % len(A)]
            for px, py in B:
                d = min(d, seg_dist(px, py, ax, ay, bx, by))
    return d if d > 0.0 else 0.0


def robot_polygon(state, robot_vertices):
    x, y, th = (float(v) for v in state)
    cs, sn = math.cos(th), math.sin(th)
    return [(x + (cs * px - sn * py), y + (sn * px + cs * py)) for px, py in robot_vertices]


def integrate(kinematics, state, action, dt, L):
    """One step of the motion models of initial_path.py:401-444 (synth.rollout's order of operations); omni takes (vx, vy)."""
    x, y, th = (float(v) for v in state)
    a0, a1 = float(action[0]), float(action[1])
    if kinematics == "omni":
        dxs, dys, dth = a0, a1, 0.0
    else:
        dxs, dys = a0 * math.cos(th), a0 * math.sin(th)
        dth = a0 * math.tan(a1) / L if kinematics == "acker" else a1
    return x + dxs * dt, y + dys * dt, th + dth * dt


def move_obstacle(row, bounds, dt):
    """Centre + v dt; a moving centre that left the rectangle is mirrored back into it and that velocity component reversed."""
    c, v = [row[0], row[1]], [row[2], row[3]]
    for a in range(2):
        c[a] = c[a] + v[a] * dt
        if v[a] != 0.0:
            lo, hi = bounds[a], bounds[2 + a]
            if c[a] < lo:
                c[a], v[a] = 2.0 * lo - c[a], -v[a]
            elif c[a] > hi:
                c[a], v[a] = 2.0 * hi - c[a], -v[a]
    return c[0], c[1], v[0], v[1]


class OracleWorld:
    """The state of B environments and the two operations of the kernels."""

    def __init__(self, cfg: dict, packed):
        self.cfg = cfg
        self.obs_begin, obs, self.vert_begin, self.vertices, self.env = (np.array(a) for a in packed)
        self.obs = obs.astype(np.float64).copy()
        self.B = len(self.obs_begin) - 1
        self.states = self.env[:, 4:7].copy()
        self.collided = np.zeros(self.B, np.int32)
        self.arrived = np.zeros(self.B, np.int32)
        self.cos_a, self.sin_a = beam_table(cfg["angle_min"], cfg["angle_max"], int(cfg["number"]))

    def scan(self, envs=None):
        """(ranges (B,R) float64, velocity (B,2,R) float64, hit (B,R), near_tie (B,R), tangent (B,R)) -- ranges before the float32
        cast."""
        R = self.cos_a.shape[0]
        envs = range(self.B) if envs is None else envs
        out = [np.zeros((self.B, R)), np.zeros((self.B, 2, R)), np.full((self.B, R), -1, np.int64), np.zeros((self.B, R), bool),
               np.zeros((self.B, R), bool)]
        for b in envs:
            o0, o1 = self.obs_begin[b], self.obs_begin[b + 1]
            circles, edges = env_boundaries(self.obs, self.vert_begin, self.vertices, o0, o1)
            sx, sy, hc, hs = sensor_ray_origin(self.states[b], self.cfg["scan_offset"])
            dx = hc * self.cos_a - hs * self.sin_a
            dy = hs * self.cos_a + hc * self.sin_a
            for i0 in range(0, R, 512):  # chunks of beams bound the (beams x boundaries) temporaries
                sl = slice(i0, min(R, i0 + 512))
                t, hit, tie, tan_ = cast(sx, sy, dx[sl], dy[sl], circles, edges, self.cfg["range_max"])
                out[0][b, sl], out[2][b, sl], out[3][b, sl], out[4][b, sl] = t, hit, tie, tan_
                for a in range(2):  # the velocity of the obstacle hit, zero on a miss
                    out[1][b, a, sl][hit >= 0] = self.obs[o0 + hit[hit >= 0], 2 + a]
        return tuple(out)

    def step(self, action):
        """action (B,2) -> (collided, arrived, clearance (B,) float64), updating the state like world_step_kernel."""
        cfg, clear = self.cfg, np.full(self.B, np.inf)
        for b in range(self.B):
            if not self.collided[b]:
                self.states[b] = integrate(cfg["kinematics"], self.states[b], action[b], cfg["step_time"], cfg.get("wheelbase"))
            x, y = self.states[b, 0], self.states[b, 1]
            gx, gy = x - self.env[b, 7], y - self.env[b, 8]
            if math.sqrt(gx * gx + gy * gy) < self.env[b, 9]:
                self.arrived[b] = 1
            robot = robot_polygon(self.states[b], cfg["robot_vertices"])
            for o in range(self.obs_begin[b], self.obs_begin[b + 1]):
                self.obs[o, :4] = move_obstacle(self.obs[o], self.env[b, :4], cfg["step_time"])
                cx, cy = self.obs[o, 0], self.obs[o, 1]
                v0, v1 = self.vert_begin[o], self.vert_begin[o + 1]
                if v1 == v0:
                    c = clearance_circle(robot, cx, cy, self.obs[o, 4])
                else:
                    c = clearance_polygon(robot, [(cx + vx, cy + vy) for vx, vy in self.vertices[v0:v1]])
                clear[b] = min(clear[b], c)
            if clear[b] <= 0.0:
                self.collided[b] = 1
        return self.collided.copy(), self.arrived.copy(), clear
