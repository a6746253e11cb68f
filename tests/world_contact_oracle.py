"""Float64 restatement of obstacle contact (nb_world_set_obstacle_contact), TEST INFRASTRUCTURE ONLY.

``ContactOracleWorld`` is ``MapMotionOracleWorld`` with the per-environment flags of ``neupan_b200.world.pack_obstacle_contact``
(``contact``).  Where a flag is 1 it adds what csrc/world_contact_kernel.cuh adds, with the kernel's operations in the kernel's order:

  * ``footprints_touch``: the contact predicate of every pair of kinds, the pair put in rank order (circle, convex, outline) first.
  * ``box``: a footprint's box, its centre plus its centre-relative box, widened by PAD; a pair is tested only when the boxes meet.
  * ``move``: the obstacles of the environment in row order (OracleWorld's step already walks them so), each taking the first of
    A (the move), B (x only), C (y only) whose footprint touches no other obstacle where it stands now, nor a blocking map, else D
    (stay); obstacle bounces per obstacle in ``obounces``, the candidate taken counted in ``otaken``.

Everything else is inherited unchanged.
"""
import math

import numpy as np

from oracle.world import clearance_outline, clearance_robots, inside_convex, inside_outline, move_obstacle, seg_dist, segs_meet
from world_map_motion_oracle import MapMotionOracleWorld

PAD = 1e-6
RANK = {"circle": 0, "convex": 1, "outline": 2}


def rel_box(shape):
    """The centre-relative box (x0, y0, x1, y1) of a footprint ("circle", r) | ("convex", rel) | ("outline", rel)."""
    kind, p = shape
    if kind == "circle":
        return -p, -p, p, p
    return float(p[:, 0].min()), float(p[:, 1].min()), float(p[:, 0].max()), float(p[:, 1].max())


def box(shape, cx, cy):
    """The footprint's box at (cx, cy), widened by PAD (the kernel's broad phase)."""
    x0, y0, x1, y1 = rel_box(shape)
    return (cx + x0) - PAD, (cy + y0) - PAD, (cx + x1) + PAD, (cy + y1) + PAD


def boxes_meet(a, b):
    return not (a[2] < b[0] or b[2] < a[0] or a[3] < b[1] or b[3] < a[1])


def _world(shape, cx, cy):
    return [(cx + float(x), cy + float(y)) for x, y in shape[1]]


def footprints_touch(sa, ca, sb, cb):
    """Do footprint sa at centre ca and sb at cb touch (clearance <= 0)?  The kernel's predicate, without the broad phase."""
    if RANK[sa[0]] > RANK[sb[0]]:
        sa, ca, sb, cb = sb, cb, sa, ca
    ka, kb = sa[0], sb[0]
    if kb == "circle":
        dx, dy = ca[0] - cb[0], ca[1] - cb[1]
        return math.sqrt(dx * dx + dy * dy) - (sa[1] + sb[1]) <= 0.0
    pb = _world(sb, *cb)
    n = len(pb)
    if ka == "circle":
        d = min(seg_dist(ca[0], ca[1], *pb[k], *pb[(k + 1) % n]) for k in range(n))
        if kb == "convex":
            return inside_convex(pb, *ca) or d - sa[1] <= 0.0
        return inside_outline(pb, *ca) or d <= sa[1]
    pa = _world(sa, *ca)
    if kb == "convex":
        return clearance_robots(pa, pb) <= 0.0
    if ka == "convex":
        return clearance_outline(pa, pb) <= 0.0
    m = len(pa)
    for k in range(m):
        for i in range(n):
            if segs_meet(pa[k], pa[(k + 1) % m], pb[i], pb[(i + 1) % n]):
                return True
    return inside_outline(pb, *pa[0]) or inside_outline(pa, *pb[0])


def touches(sa, ca, sb, cb):
    """The broad phase, then footprints_touch."""
    return boxes_meet(box(sa, *ca), box(sb, *cb)) and footprints_touch(sa, ca, sb, cb)


class ContactOracleWorld(MapMotionOracleWorld):
    def __init__(self, cfg: dict, packed, behaviors=None, seed: int = 0, *, contact=None, **kw):
        super().__init__(cfg, packed, behaviors, seed, **kw)
        O = len(self.obs)
        self.contact = np.zeros(self.B, np.int32) if contact is None else np.asarray(contact, np.int32).copy()
        self.obounces = np.zeros(O, np.int32)
        self.otaken = dict(B=0, C=0, D=0)
        self.shapes = [self.shape(o) for o in range(O)]
        self.rboxes = np.array([rel_box(s) for s in self.shapes]).reshape(-1, 4)

    def touches_others(self, b, o, cx, cy):
        """Does obstacle o at (cx, cy) touch another obstacle of environment b where it stands now?"""
        o0, o1 = self.obs_begin[b], self.obs_begin[b + 1]
        rb = self.rboxes[o0:o1]
        c = self.obs[o0:o1, :2]
        x0, y0, x1, y1 = ((cx + self.rboxes[o, 0]) - PAD, (cy + self.rboxes[o, 1]) - PAD, (cx + self.rboxes[o, 2]) + PAD,
                          (cy + self.rboxes[o, 3]) + PAD)
        meet = ~((x1 < (c[:, 0] + rb[:, 0]) - PAD) | ((c[:, 0] + rb[:, 2]) + PAD < x0) | (y1 < (c[:, 1] + rb[:, 1]) - PAD)
                 | ((c[:, 1] + rb[:, 3]) + PAD < y0))
        meet[o - o0] = False
        sa = self.shapes[o]
        return any(footprints_touch(sa, (cx, cy), self.shapes[p], (float(self.obs[p, 0]), float(self.obs[p, 1])))
                   for p in np.flatnonzero(meet) + o0)

    def move(self, b, o):
        """MapMotionOracleWorld.move, or where environment b has obstacle contact the sequential move rule."""
        if not self.contact[b]:
            return super().move(b, o)
        row = self.obs[o]
        x, y, moves = float(row[0]), float(row[1]), row[2] != 0.0 or row[3] != 0.0
        cx, cy, vx, vy = move_obstacle(row, self.env[b, :4], self.cfg["step_time"])
        blocks = bool(self.block[b])
        take, obs_a, map_a = 0, False, False
        if moves:
            for take, (px, py) in enumerate(((cx, cy), (cx, y), (x, cy))):
                to = self.touches_others(b, o, px, py)
                tm = blocks and (take == 0 or not to) and self.touches(b, o, px, py)
                if take == 0:
                    obs_a, map_a = to, tm
                if not to and not tm:
                    break
            else:
                take = 3
        if take == 1:
            cy, vy = y, -vy
        elif take == 2:
            cx, vx = x, -vx
        elif take == 3:
            cx, cy, vx, vy = x, y, -vx, -vy
        self.obs[o, :4] = cx, cy, vx, vy
        if take:
            self.otaken["BCD"[take - 1]] += 1
        if obs_a:
            self.obounces[o] += 1
        if blocks:
            if map_a:
                self.bounces[o] += 1
            self.bounced[o] = map_a

    def moving(self):
        """(O,) bool: obstacles that can move (v != 0, or reactive)."""
        return (self.beh[:, 0] == 1.0) | np.any(self.obs[:, 2:4] != 0.0, 1)

    def touching_pairs(self, movers=None):
        """Pairs (o, p), o < p, of one environment with the flag set that touch now, at least one of them a mover."""
        movers = self.moving() if movers is None else movers
        out = []
        for b in np.flatnonzero(self.contact):
            o0, o1 = self.obs_begin[b], self.obs_begin[b + 1]
            c, rb = self.obs[o0:o1, :2], self.rboxes[o0:o1]
            lo, hi = (c + rb[:, :2]) - PAD, (c + rb[:, 2:]) + PAD
            meet = ~((hi[:, None, 0] < lo[None, :, 0]) | (hi[None, :, 0] < lo[:, None, 0]) | (hi[:, None, 1] < lo[None, :, 1])
                     | (hi[None, :, 1] < lo[:, None, 1]))
            meet &= movers[o0:o1, None] | movers[None, o0:o1]
            for o, p in zip(*np.nonzero(np.triu(meet, 1))):
                if footprints_touch(self.shapes[o0 + o], tuple(c[o]), self.shapes[o0 + p], tuple(c[p])):
                    out.append((int(o0 + o), int(o0 + p)))
        return out

    def move_all(self):
        """The obstacle motion of one step alone (no robots): every environment's obstacles in row order."""
        for b in range(self.B):
            for o in range(self.obs_begin[b], self.obs_begin[b + 1]):
                self.move(b, o)
