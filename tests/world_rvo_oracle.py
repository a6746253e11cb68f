"""CPU restatement of the world's reactive obstacles (behaviour kind 1 of nb_world_set_behaviors), on top of
tests/world_outline_oracle.py.

Float64, the same operations in the same order as world_rvo_kernel in csrc/world_rvo_kernel.cuh (Python rounds every product, sum,
quotient and square root separately, as the kernel does with __dmul_rn / __dadd_rn / __dsub_rn / __ddiv_rn / __dsqrt_rn).
``OracleWorld`` here takes the packed scenes of world_outline_oracle.OracleWorld plus the (O, 13) behaviour rows and a seed; its
``step`` first chooses every reactive obstacle's velocity from the states at the start of the step (``rvo``), then runs the parent's
step unchanged.  The one difference from the kernel is the robot's velocity: libm's cos / sin here, CUDA's sincos there.  ``rvo``
therefore also reports, per obstacle, the smallest decision margin that involved the robot (cone-edge cross products of its cone,
and in the penalty pass the gap between the best and the second-best penalty), so that a test can tell a libm difference from a bug.

The goal draws use SplitMix64 in numpy uint64 arithmetic: output n of the generator seeded with s is mix(s + (n + 1) gamma).
"""
import math

import numpy as np

from oracle import world as ow
import world_outline_oracle as wo

BEH_COLS = 13
MAX_AXIS = 64
GAMMA = np.uint64(0x9E3779B97F4A7C15)


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


def inside(cn, vx, vy):
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


class OracleWorld(wo.OracleWorld):
    """world_outline_oracle.OracleWorld with obstacle behaviours: ``behaviors`` (O, 13) rows of pack_behaviors (None: every obstacle
    keeps a constant velocity), ``seed`` the goal draws' seed."""

    def __init__(self, cfg: dict, packed, behaviors=None, seed: int = 0):
        super().__init__(cfg, packed)
        O = len(self.obs)
        self.beh = np.zeros((O, BEH_COLS)) if behaviors is None else np.array(behaviors, np.float64).reshape(O, BEH_COLS)
        self.seed = int(seed)
        self.radius = np.array([radius_of(self.obs, self.vert_begin, self.vertices, o) for o in range(O)])
        self.robot_r = max(math.sqrt(x * x + y * y) for x, y in np.asarray(cfg["robot_vertices"], np.float64))
        self.goal = np.zeros((O, 2))
        self.draws = np.zeros(O, np.int32)
        for b in range(self.B):
            for o in range(self.obs_begin[b], self.obs_begin[b + 1]):
                if self.beh[o, 0] != 1.0:
                    continue
                if math.isnan(self.beh[o, 7]):
                    self.goal[o] = draw_goal(self.seed, b, o - self.obs_begin[b], 0, self.env[b, :4])
                    self.draws[o] = 1
                else:
                    self.goal[o] = self.beh[o, 7:9]

    def robot_velocity(self, b, action):
        if self.collided[b]:
            return 0.0, 0.0
        a0, a1 = float(action[b][0]), float(action[b][1])
        if self.cfg["kinematics"] == "omni":
            return a0, a1
        th = float(self.states[b, 2])
        return a0 * math.cos(th), a0 * math.sin(th)

    def choose(self, b, i, rows, robot_row):
        """Obstacle i of environment b: (vx, vy, goal, draws, robot_margin) from the rows (cx, cy, vx, vy, r) of the environment's
        obstacles at the start of the step and the robot's row."""
        o0 = self.obs_begin[b]
        o = o0 + i
        beh, env = self.beh[o], self.env[b]
        n = len(rows)
        allrows = rows + [robot_row]
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
        for j in range(n + 1):
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
            if j == n:  # the robot's cone: how far each candidate is from either edge decision
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
        if any(j == n for j, _ in cones) and len(pen) > 1:
            p = np.sort(pen)
            margin = min(margin, float(p[1] - p[0]) if np.isfinite(p[1]) else math.inf)
        return float(ux[q]), float(uy[q]), (gx, gy), draws, margin

    def rvo(self, action, envs=None):
        """Chooses every reactive obstacle's velocity (writing it into its row) from the states at the start of the step, in the
        environments ``envs`` (default all).  Returns the per-obstacle robot margins (inf where the robot was not a neighbour or the
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
            rvx, rvy = self.robot_velocity(b, action)
            robot_row = (float(self.states[b, 0]), float(self.states[b, 1]), rvx, rvy, self.robot_r)
            for o in range(o0, o1):
                if self.beh[o, 0] == 1.0:
                    new[o] = self.choose(b, o - o0, rows, robot_row)
        for o, (vx, vy, g, d, m) in new.items():
            self.obs[o, 2], self.obs[o, 3] = vx, vy
            self.goal[o] = g
            self.draws[o] = d
            margins[o] = m
        return margins

    def step(self, action):
        """rvo, then world_outline_oracle.OracleWorld.step.  Also keeps the robot margins of the step in ``self.margins``."""
        self.margins = self.rvo(action)
        return super().step(action)
