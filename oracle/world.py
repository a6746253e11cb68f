"""CPU restatement of the batched 2-D world (TEST INFRASTRUCTURE ONLY, like the rest of oracle/).

Float64, the same operations in the same order as csrc/world_kernel.cuh and csrc/world_rvo_kernel.cuh (which round every product,
sum, quotient and square root separately, no FMA), so that the kernels agree with it to the last bit wherever their inputs agree;
the only differences come from CUDA's sin / cos / tan vs libm (the robots' integration, bodies and velocities).  ``OracleWorld`` takes
the packed arrays of ``neupan_b200.world.pack_scenes`` (5) or ``pack_scenes_ex`` (6, the last one the obstacle kinds), optionally the
(O, 13) behaviour rows of ``pack_behaviors`` with their seed and the (B K, 6) robot rows of ``pack_fleet`` (without them: the env
rows' start and goal, K = 1), and a config dict:

    kinematics ("diff" | "acker" | "omni"), step_time, wheelbase, angle_min, angle_max, range_max, number (R),
    scan_offset (3,), robot_vertices (n, 2) in the robot frame.

Robot k of environment b is row n = b K + k of every per-robot array.

Geometry:
  * ray / circle: |s + t d - c|^2 = r^2 with |d| = 1:  t = -b -+ sqrt(b^2 - c'),  b = (s - c).d,  c' = |s - c|^2 - r^2
  * ray / segment a->b:  s + t d = a + u e,  e = b - a,  w = a - s:  t = (w x e) / (d x e),  u = (w x d) / (d x e),  0 <= u <= 1
  * the range is the smallest t > 0 over all boundaries (equal t: the lower index, obstacles 0..O_b - 1 then robot j as O_b + j);
    none below range_max: range_max, hit -1.  With K > 1 a beam also crosses the bodies of the other robots, never its own.
  * clearance robot polygon <-> circle: distance from the centre to the polygon (0 inside) - r;  <-> convex polygon (and robot <->
    robot): 0 unless an edge normal of either polygon separates them (SAT), else the smallest vertex-edge distance;  <-> outline
    (kind 1, any simple polygon): 0 when an edge meets a robot edge or one lies inside the other, else the vertex-edge distances;
    clamped at 0
Step: reactive obstacles choose their velocities first (``rvo``: every robot a neighbour row, after the obstacles); then Jacobi:
every robot that has not collided integrates from the state at the start of the step, the obstacles move once, and each robot's
clearance is the minimum over the obstacles and the other robots.

Reactive obstacles (behaviour kind 1): csrc/world_rvo_kernel.cuh states the rule.  ``rvo`` also reports, per obstacle, the smallest
decision margin that involved a robot (cone-edge cross products of a robot's cone, and in the penalty pass the gap between the best
and the second-best penalty), so that a test can tell a libm difference from a bug.  The goal draws use SplitMix64 in numpy uint64
arithmetic: output n of the generator seeded with s is mix(s + (n + 1) gamma).
"""
import math

import numpy as np

KIN = {"diff": 0, "acker": 1, "omni": 2}
BEH_COLS = 13
MAX_AXIS = 64
GAMMA = np.uint64(0x9E3779B97F4A7C15)


# ---- lidar ---------------------------------------------------------------------------------------------------------------------

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


# ---- clearance -----------------------------------------------------------------------------------------------------------------

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


def _vertex_edge_distance(P, Q):
    """The smallest distance from a vertex of Q to an edge of P, then from a vertex of P to an edge of Q (the kernels' order)."""
    d = math.inf
    for A, B in ((P, Q), (Q, P)):
        for k in range(len(A)):
            (ax, ay), (bx, by) = A[k], A[(k + 1) % len(A)]
            for px, py in B:
                d = min(d, seg_dist(px, py, ax, ay, bx, by))
    return d


def inside_convex(robot, x, y):
    """The circle branch's test: (x, y) is not strictly outside the convex polygon (the edge cross products do not take both
    signs)."""
    pos = neg = False
    n = len(robot)
    for k in range(n):
        (ax, ay), (bx, by) = robot[k], robot[(k + 1) % n]
        cr = (bx - ax) * (y - ay) - (by - ay) * (x - ax)
        pos, neg = pos or cr > 0.0, neg or cr < 0.0
    return not (pos and neg)


def clearance_circle(robot, cx, cy, r):
    """Robot polygon (list of world vertices) <-> circle."""
    n = len(robot)
    d = min(seg_dist(cx, cy, *robot[k], *robot[(k + 1) % n]) for k in range(n))
    c = 0.0 if inside_convex(robot, cx, cy) else d - r  # the centre inside the robot: overlap
    return c if c > 0.0 else 0.0


def clearance_polygon(robot, poly):
    """Robot polygon <-> convex polygon (lists of world vertices)."""
    if not (_separated(robot, poly) or _separated(poly, robot)):
        return 0.0
    d = _vertex_edge_distance(poly, robot)
    return d if d > 0.0 else 0.0


def clearance_robots(P, Q):
    """Robot <-> robot (lists of world vertices): the convex branch, which evaluates both SAT orders and both distance directions,
    so it is symmetric in P and Q."""
    return clearance_polygon(P, Q)


def _in_box(a, b, p):
    return min(a[0], b[0]) <= p[0] <= max(a[0], b[0]) and min(a[1], b[1]) <= p[1] <= max(a[1], b[1])


def segs_meet(p, q, a, b):
    """Do the closed segments p-q and a-b intersect or touch?"""
    ex, ey, fx, fy = b[0] - a[0], b[1] - a[1], q[0] - p[0], q[1] - p[1]
    d1 = ex * (p[1] - a[1]) - ey * (p[0] - a[0])
    d2 = ex * (q[1] - a[1]) - ey * (q[0] - a[0])
    d3 = fx * (a[1] - p[1]) - fy * (a[0] - p[0])
    d4 = fx * (b[1] - p[1]) - fy * (b[0] - p[0])
    if ((d1 > 0.0 and d2 < 0.0) or (d1 < 0.0 and d2 > 0.0)) and ((d3 > 0.0 and d4 < 0.0) or (d3 < 0.0 and d4 > 0.0)):
        return True
    return ((d1 == 0.0 and _in_box(a, b, p)) or (d2 == 0.0 and _in_box(a, b, q)) or (d3 == 0.0 and _in_box(p, q, a))
            or (d4 == 0.0 and _in_box(p, q, b)))


def inside_outline(poly, x, y):
    """Even-odd test of (x, y) against the polygon (list of (x, y)): an edge straddling the horizontal line through the point
    toggles it when it crosses that line to the point's right (the sign of edge x (point - edge start))."""
    n, res = len(poly), False
    for k in range(n):
        (ax, ay), (bx, by) = poly[k], poly[(k + 1) % n]
        if (ay > y) != (by > y):
            c = (bx - ax) * (y - ay) - (by - ay) * (x - ax)
            if (c > 0.0) if by > ay else (c < 0.0):
                res = not res
    return res


def clearance_outline(robot, poly):
    """Robot polygon (convex) <-> outline (any simple polygon), lists of world vertices: 0 when an outline edge meets a robot edge,
    robot vertex 0 lies inside the outline or outline vertex 0 inside the robot; else the smallest vertex-edge distance both ways,
    in clearance_polygon's order."""
    nr, nv = len(robot), len(poly)
    for k in range(nv):
        for i in range(nr):
            if segs_meet(robot[i], robot[(i + 1) % nr], poly[k], poly[(k + 1) % nv]):
                return 0.0
    if inside_outline(poly, *robot[0]) or inside_convex(robot, *poly[0]):
        return 0.0
    d = _vertex_edge_distance(poly, robot)
    return d if d > 0.0 else 0.0


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


# ---- motion --------------------------------------------------------------------------------------------------------------------

def robot_polygon(state, robot_vertices):
    x, y, th = (float(v) for v in state)
    cs, sn = math.cos(th), math.sin(th)
    return [(x + (cs * px - sn * py), y + (sn * px + cs * py)) for px, py in robot_vertices]


def robot_velocity(kinematics, action, th):
    """World-frame translation rate of the action at heading th: diff / acker v (cos th, sin th), omni (vx, vy)."""
    a0, a1 = float(action[0]), float(action[1])
    return (a0, a1) if kinematics == "omni" else (a0 * math.cos(th), a0 * math.sin(th))


def integrate(kinematics, state, action, dt, L):
    """One step of the motion models of initial_path.py:401-444 (synth.rollout's order of operations); omni takes (vx, vy)."""
    x, y, th = (float(v) for v in state)
    a0, a1 = float(action[0]), float(action[1])
    dxs, dys = robot_velocity(kinematics, action, th)
    dth = 0.0 if kinematics == "omni" else (a0 * math.tan(a1) / L if kinematics == "acker" else a1)
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


# ---- reactive obstacles --------------------------------------------------------------------------------------------------------

def splitmix64_mix(z):
    z = np.uint64(z)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def splitmix64_at(s, n):
    """Output n (0-based) of SplitMix64 seeded with s."""
    with np.errstate(over="ignore"):
        return splitmix64_mix(np.uint64(s) + np.uint64(n + 1) * GAMMA)


def rvo_key(seed, b, i):
    """The stream of obstacle i (index within its environment) of environment b."""
    with np.errstate(over="ignore"):
        s = splitmix64_mix(np.uint64(seed) + GAMMA)
    return splitmix64_mix(s ^ np.uint64((int(b) << 32) | int(i)))


def u01(x):
    return float(np.uint64(x) >> np.uint64(11)) * 2.0 ** -53


def draw_goal(seed, b, i, n, bounds):
    """Draw n of obstacle i of environment b: a point of the rectangle (xmin, ymin, xmax, ymax)."""
    key = rvo_key(seed, b, i)
    gx = bounds[0] + u01(splitmix64_at(key, 2 * n)) * (bounds[2] - bounds[0])
    gy = bounds[1] + u01(splitmix64_at(key, 2 * n + 1)) * (bounds[3] - bounds[1])
    return gx, gy


def cone(ci, vi, ri, cj, vj, rj):
    """The RVO cone of neighbour j seen from i: (apex, left edge, right edge), trigonometry-free."""
    px, py = cj[0] - ci[0], cj[1] - ci[1]
    D = math.sqrt(px * px + py * py)
    R = ri + rj
    Dp = D if D > R else R
    sa = R / Dp
    ca = math.sqrt(Dp * Dp - R * R) / Dp
    ux, uy = px / D, py / D
    apex = (0.5 * (vi[0] + vj[0]), 0.5 * (vi[1] + vj[1]))
    left = (ux * ca - uy * sa, ux * sa + uy * ca)
    right = (ux * ca + uy * sa, uy * ca - ux * sa)
    return apex, left, right


def cone_trig(ci, vi, ri, cj, vj, rj):
    """IR-SIM's construction of the same cone, with atan2 / asin / cos / sin."""
    px, py = cj[0] - ci[0], cj[1] - ci[1]
    D = math.sqrt(px * px + py * py)
    R = ri + rj
    Dp = max(D, R)
    ang, half = math.atan2(py, px), math.asin(R / Dp)
    apex = ((vi[0] + vj[0]) / 2, (vi[1] + vj[1]) / 2)
    return apex, (math.cos(ang + half), math.sin(ang + half)), (math.cos(ang - half), math.sin(ang - half))


def cross(a, bx, by):
    return a[0] * by - a[1] * bx


def inside_cone(cn, vx, vy):
    """between_vector: w = v - apex lies between the cone's edges (closed)."""
    apex, left, right = cn
    wx, wy = vx - apex[0], vy - apex[1]
    return cross(left, wx, wy) <= 0.0 and cross(right, wx, wy) >= 0.0


def axis_count(lo, hi, grid):
    if not hi > lo:
        return 0
    n = math.ceil((hi - lo) / grid)
    return n if n < MAX_AXIS else MAX_AXIS


def radius_of(obs, vert_begin, vertices, o):
    """A circle's radius, or a polygon's circumradius about its centre."""
    v0, v1 = vert_begin[o], vert_begin[o + 1]
    r = float(obs[o, 4]) if v0 == v1 else 0.0
    for x, y in vertices[v0:v1]:
        r = max(r, math.sqrt(x * x + y * y))
    return r


# ---- the world -----------------------------------------------------------------------------------------------------------------

class OracleWorld:
    """The state of B environments of K robots each and the operations of the kernels.  ``behaviors``: (O, 13) rows of
    pack_behaviors (None: every obstacle keeps a constant velocity); ``seed``: the goal draws' seed; ``fleet``: (B K, 6) rows
    [start x, y, theta, goal x, y, threshold] (None: the env rows, K = 1)."""

    def __init__(self, cfg: dict, packed, behaviors=None, seed: int = 0, *, fleet=None, K: int = 1):
        self.cfg = cfg
        self.obs_begin, obs, self.vert_begin, self.vertices, self.env = (np.array(a) for a in packed[:5])
        self.obs = obs.astype(np.float64).copy()
        O = len(self.obs)
        self.kind = np.array(packed[5]) if len(packed) > 5 else np.zeros(O, np.int32)
        self.B, self.K = len(self.obs_begin) - 1, int(K)
        self.N = self.B * self.K
        fleet = self.env[:, 4:10] if fleet is None else np.asarray(fleet, np.float64).reshape(self.N, 6)
        self.states = fleet[:, :3].copy()
        self.fgoal = fleet[:, 3:6].copy()
        self.collided = np.zeros(self.N, np.int32)
        self.arrived = np.zeros(self.N, np.int32)
        self.fvel = np.zeros((self.N, 2))  # world-frame velocity of each robot's last step
        self.robot_clear = np.full(self.N, np.inf)  # the part of the last step's clearance that comes from the other robots
        self.rv = np.asarray(cfg["robot_vertices"], np.float64)
        self.cos_a, self.sin_a = beam_table(cfg["angle_min"], cfg["angle_max"], int(cfg["number"]))
        self.beh = np.zeros((O, BEH_COLS)) if behaviors is None else np.array(behaviors, np.float64).reshape(O, BEH_COLS)
        self.seed = int(seed)
        self.radius = np.array([radius_of(self.obs, self.vert_begin, self.vertices, o) for o in range(O)])
        self.robot_r = max(math.sqrt(x * x + y * y) for x, y in self.rv)
        self.goal = np.zeros((O, 2))
        self.draws = np.zeros(O, np.int32)
        self.margins = np.full(O, math.inf)
        self.paths = {}
        for b in range(self.B):
            for o in range(self.obs_begin[b], self.obs_begin[b + 1]):
                if self.beh[o, 0] != 1.0:
                    continue
                if math.isnan(self.beh[o, 7]):
                    self.goal[o] = draw_goal(self.seed, b, o - self.obs_begin[b], 0, self.env[b, :4])
                    self.draws[o] = 1
                else:
                    self.goal[o] = self.beh[o, 7:9]

    def bodies(self, b):
        return [robot_polygon(self.states[b * self.K + j], self.rv) for j in range(self.K)]

    # ---- scan ----
    def scan(self, envs=None):
        """(ranges (N,R) float64, velocity (N,2,R) float64, hit (N,R), near_tie (N,R), tangent (N,R)) -- ranges before the float32
        cast.  A beam of robot k casts against the environment's obstacles and, with K > 1, the edges of the other robots' bodies,
        ids O_b + j; a robot hit reports that robot's velocity from its last step."""
        R, K = self.cos_a.shape[0], self.K
        envs = range(self.B) if envs is None else envs
        out = [np.zeros((self.N, R)), np.zeros((self.N, 2, R)), np.full((self.N, R), -1, np.int64), np.zeros((self.N, R), bool),
               np.zeros((self.N, R), bool)]
        for b in envs:
            o0, o1 = self.obs_begin[b], self.obs_begin[b + 1]
            nobs = o1 - o0
            circles, edges = env_boundaries(self.obs, self.vert_begin, self.vertices, o0, o1)
            bodies = self.bodies(b) if K > 1 else []
            for k in range(K):
                n = b * K + k
                redges = [(*body[v], *body[(v + 1) % len(body)], nobs + j) for j, body in enumerate(bodies) if j != k for v in range(len(body))]
                E = np.concatenate([edges, np.array(redges, np.float64).reshape(-1, 5)])
                sx, sy, hc, hs = sensor_ray_origin(self.states[n], self.cfg["scan_offset"])
                dx = hc * self.cos_a - hs * self.sin_a
                dy = hs * self.cos_a + hc * self.sin_a
                for i0 in range(0, R, 512):  # chunks of beams bound the (beams x boundaries) temporaries
                    sl = slice(i0, min(R, i0 + 512))
                    t, hit, tie, tan_ = cast(sx, sy, dx[sl], dy[sl], circles, E, self.cfg["range_max"])
                    out[0][n, sl], out[2][n, sl], out[3][n, sl], out[4][n, sl] = t, hit, tie, tan_
                    ob, rb = (hit >= 0) & (hit < nobs), hit >= nobs
                    for a in range(2):  # the velocity of the object hit, zero on a miss
                        out[1][n, a, sl][ob] = self.obs[o0 + hit[ob], 2 + a]
                        out[1][n, a, sl][rb] = self.fvel[b * K + hit[rb] - nobs, a]
        return tuple(out)

    # ---- reactive obstacles ----
    def robot_rows(self, b, action):
        """The neighbour rows (x, y, vx, vy, r) of the environment's robots: velocity 0 once collided, else this step's action's."""
        rows = []
        for n in range(b * self.K, (b + 1) * self.K):
            v = (0.0, 0.0) if self.collided[n] else robot_velocity(self.cfg["kinematics"], action[n], float(self.states[n, 2]))
            rows.append((float(self.states[n, 0]), float(self.states[n, 1]), v[0], v[1], self.robot_r))
        return rows

    def choose(self, b, i, rows, robot_rows):
        """Obstacle i of environment b: (vx, vy, goal, draws, robot_margin) from the rows (cx, cy, vx, vy, r) of the environment's
        obstacles at the start of the step and the rows of its robots (after the obstacles); the margin covers every robot's cone."""
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
                gx, gy = draw_goal(self.seed, b, i, draws, env[:4])
                draws += 1
                dx, dy = gx - cx, gy - cy
                dist = math.sqrt(dx * dx + dy * dy)
            else:
                self.paths[o] = "parked"
                return 0.0, 0.0, (gx, gy), draws, margin
        desx = desy = 0.0
        if dist > 0.0:
            desx, desy = (beh[5] * dx) / dist, (beh[5] * dy) / dist
        cones = []  # (neighbour index, cone)
        for j in range(len(allrows)):
            if j == i:
                continue
            px, py = allrows[j][0] - cx, allrows[j][1] - cy
            D = math.sqrt(px * px + py * py)
            if D > 0.0 and D <= beh[10]:
                cones.append((j, cone((cx, cy), (vx, vy), ri, allrows[j][:2], allrows[j][2:4], allrows[j][4])))
        grid, ms = beh[11], beh[12]
        lxa, lxb, hxa, hxb = vx - beh[3], -beh[1], vx + beh[3], beh[1]
        lya, lyb, hya, hyb = vy - beh[3], -beh[2], vy + beh[3], beh[2]
        lox, hix = (lxa if lxa > lxb else lxb), (hxa if hxa < hxb else hxb)
        loy, hiy = (lya if lya > lyb else lyb), (hya if hya < hyb else hyb)
        nx, ny = axis_count(lox, hix, grid), axis_count(loy, hiy, grid)
        # the candidates as numpy arrays: elementwise float64 operations, each rounded on its own like the scalar code
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
            if j >= n:  # a robot's cone: how far each candidate is from either edge decision
                margin = min(margin, float(np.minimum(np.abs(c1), np.abs(c2)).min()))
        ex, ey = ux - desx, uy - desy
        key = np.sqrt(ex * ex + ey * ey)
        if out.any():
            q = int(np.flatnonzero(out)[np.argmin(key[out])])  # the first of equal keys: the lower index
            self.paths[o] = "outside"
            return float(ux[q]), float(uy[q]), (gx, gy), draws, margin
        tmin = np.full(len(k), np.inf)  # every candidate inside a cone: the smallest penalty
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
        """Chooses every reactive obstacle's velocity (writing it into its row) from the states at the start of the step, in the
        environments ``envs`` (default all).  Returns the per-obstacle robot margins (inf where no robot was a neighbour or the
        obstacle is not reactive); ``self.paths`` maps each reactive obstacle to how its velocity was chosen ("outside", "penalty",
        "none": no candidate, "parked")."""
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
                    new[o] = self.choose(b, o - o0, rows, robots)
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
            return clearance_circle(body, cx, cy, self.obs[o, 4])
        poly = [(cx + vx, cy + vy) for vx, vy in self.vertices[v0:v1]]
        return clearance_outline(body, poly) if self.kind[o] == 1 else clearance_polygon(body, poly)

    def step(self, action, rvo=True):
        """action (N,2) -> (collided, arrived, clearance (N,) float64), updating the state like world_step_kernel; first the
        reactive obstacles' choice (``rvo=False`` skips it: a teacher-forced test runs it separately), whose robot margins stay in
        ``self.margins``."""
        if rvo:
            self.margins = self.rvo(action)
        cfg, K = self.cfg, self.K
        clear = np.full(self.N, np.inf)
        self.robot_clear = np.full(self.N, np.inf)
        vel = np.zeros((self.N, 2))
        for n in range(self.N):
            if not self.collided[n]:
                vel[n] = robot_velocity(cfg["kinematics"], action[n], float(self.states[n, 2]))
                self.states[n] = integrate(cfg["kinematics"], self.states[n], action[n], cfg["step_time"], cfg.get("wheelbase"))
            gx, gy = self.states[n, 0] - self.fgoal[n, 0], self.states[n, 1] - self.fgoal[n, 1]
            if math.sqrt(gx * gx + gy * gy) < self.fgoal[n, 2]:
                self.arrived[n] = 1
        for b in range(self.B):
            o0, o1 = self.obs_begin[b], self.obs_begin[b + 1]
            for o in range(o0, o1):
                self.obs[o, :4] = move_obstacle(self.obs[o], self.env[b, :4], cfg["step_time"])
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
