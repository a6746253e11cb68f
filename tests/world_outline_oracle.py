"""CPU restatement of the world's outline obstacles (kind 1 of nb_world_set_scenes_ex), on top of oracle/world.py.

Float64, the same operations in the same order as world_outline_clearance in csrc/world_kernel.cuh (Python rounds every product
and sum separately, as the kernel does with __dmul_rn / __dadd_rn / __dsub_rn).  oracle/world.py stays the reference for circles
and convex polygons; ``OracleWorld`` here takes the packed arrays of ``pack_scenes`` (5) or ``pack_scenes_ex`` (6, the last one
the kinds) and sends kind-1 obstacles to ``clearance_outline``.  The scan needs nothing new: an outline's edges are cast like a
convex polygon's.
"""
import math

import numpy as np

from oracle import world as ow


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


def inside(poly, x, y):
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


def clearance_outline(robot, poly):
    """Robot polygon (convex) <-> outline (any simple polygon), lists of world vertices: 0 when an outline edge meets a robot edge,
    robot vertex 0 lies inside the outline or outline vertex 0 inside the robot; else the smallest vertex-edge distance both ways,
    in clearance_polygon's order."""
    nr, nv = len(robot), len(poly)
    for k in range(nv):
        for i in range(nr):
            if segs_meet(robot[i], robot[(i + 1) % nr], poly[k], poly[(k + 1) % nv]):
                return 0.0
    if inside(poly, *robot[0]) or inside_convex(robot, *poly[0]):
        return 0.0
    d = math.inf
    for A, B in ((poly, robot), (robot, poly)):  # vertices of B against the edges of A
        for k in range(len(A)):
            (ax, ay), (bx, by) = A[k], A[(k + 1) % len(A)]
            for px, py in B:
                d = min(d, ow.seg_dist(px, py, ax, ay, bx, by))
    return d if d > 0.0 else 0.0


class OracleWorld(ow.OracleWorld):
    """oracle.world.OracleWorld with outlines: ``packed`` is the 5 arrays of pack_scenes or the 6 of pack_scenes_ex."""

    def __init__(self, cfg: dict, packed):
        super().__init__(cfg, packed[:5])
        self.kind = np.array(packed[5]) if len(packed) > 5 else np.zeros(len(self.obs), np.int32)

    def step(self, action):
        """world_step_kernel's step with the kind-1 branch (the rest as oracle.world.OracleWorld.step)."""
        cfg, clear = self.cfg, np.full(self.B, np.inf)
        for b in range(self.B):
            if not self.collided[b]:
                self.states[b] = ow.integrate(cfg["kinematics"], self.states[b], action[b], cfg["step_time"], cfg.get("wheelbase"))
            x, y = self.states[b, 0], self.states[b, 1]
            gx, gy = x - self.env[b, 7], y - self.env[b, 8]
            if math.sqrt(gx * gx + gy * gy) < self.env[b, 9]:
                self.arrived[b] = 1
            robot = ow.robot_polygon(self.states[b], cfg["robot_vertices"])
            for o in range(self.obs_begin[b], self.obs_begin[b + 1]):
                self.obs[o, :4] = ow.move_obstacle(self.obs[o], self.env[b, :4], cfg["step_time"])
                cx, cy = self.obs[o, 0], self.obs[o, 1]
                v0, v1 = self.vert_begin[o], self.vert_begin[o + 1]
                if v1 == v0:
                    c = ow.clearance_circle(robot, cx, cy, self.obs[o, 4])
                else:
                    poly = [(cx + vx, cy + vy) for vx, vy in self.vertices[v0:v1]]
                    c = clearance_outline(robot, poly) if self.kind[o] == 1 else ow.clearance_polygon(robot, poly)
                clear[b] = min(clear[b], c)
            if clear[b] <= 0.0:
                self.collided[b] = 1
        return self.collided.copy(), self.arrived.copy(), clear
