"""Actuation limits, motion noise and lidar range noise of the batched world (csrc/world_kernel.cuh, "Actuation limits and noise"),
restated in float64 Python with the kernels' operations in the kernels' order.  It composes with every world oracle: ``Actuation.apply``
turns the step's actions into the velocities the robots integrate (pass them to ``step(u, rvo=False)`` after ``rvo(action)``, since
reactive obstacles see the action as given), and ``lidar_noise`` turns an oracle scan's float64 ranges into the noisy ones."""
import math

import numpy as np

from oracle.world import rvo_key, splitmix64_at, splitmix64_mix, u01

TAG_MOTION = 0x6D6F74696F6E0001
TAG_LIDAR = 0x6C69646172000002
TWO_PI = 6.283185307179586
DEFAULT_ROW = (-math.inf, -math.inf, math.inf, math.inf, math.inf, math.inf, 0.0, 0.0, 0.0, 0.0)


def noise_key(seed, tag, e, k, n):
    """The noise stream of robot k of environment (scene) e at step n under a domain tag."""
    return splitmix64_at(splitmix64_mix(rvo_key(seed, e, k) ^ np.uint64(tag)), int(n))


def normal(key, j):
    """Draw j of a step's stream: Box-Muller from outputs 2j and 2j + 1."""
    u1, u2 = u01(splitmix64_at(key, 2 * j)), u01(splitmix64_at(key, 2 * j + 1))
    return math.sqrt(-2.0 * math.log(1.0 - u1)) * math.cos(TWO_PI * u2)


def normals(key, j):
    """``normal`` for an array of draw numbers j at once (numpy's log and cos: for statistics)."""
    j = np.asarray(j, np.uint64)
    with np.errstate(over="ignore"):
        u1 = (splitmix64_at(key, 2 * j) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
        u2 = (splitmix64_at(key, 2 * j + np.uint64(1)) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    return np.sqrt(-2.0 * np.log(1.0 - u1)) * np.cos(TWO_PI * u2)


def limit(a, prev, row, dt):
    """One component: the command after the bounds and the rate limit (row: vel_min, vel_max, acce of that component)."""
    vmin, vmax, acce = row
    r = acce * dt
    lo, hi = max(vmin, prev - r), min(vmax, prev + r)
    return min(max(a, lo), hi)


class Actuation:
    """Per-type rows (T, 10) [vel_min (2), vel_max (2), acce (2), alpha (4)] (neupan_b200.world.pack_actuation), the motion seed and
    every robot row's cmd_prev."""

    def __init__(self, rows, seed, N, dt):
        self.rows = np.asarray(rows, np.float64).reshape(-1, 10)
        self.seed, self.dt = int(seed), float(dt)
        self.cmd = np.zeros((N, 2))

    def row(self, t):
        return self.rows[t] if t < len(self.rows) else np.asarray(DEFAULT_ROW)

    def apply(self, action, collided, K, rtype=None, n=0, scene=None):
        """(N, 2) float64 velocities to integrate from the (float32) actions; updates cmd_prev.  Row q's robot is robot q mod K of
        environment q // K (``scene``: the scene of each row's environment in episode mode); ``n`` the step (an int, or per row)."""
        N = len(self.cmd)
        u = np.zeros((N, 2))
        steps = np.broadcast_to(np.asarray(n, np.int64), (N,))
        for q in range(N):
            if collided[q]:
                self.cmd[q] = 0.0
                continue
            A = self.row(0 if rtype is None else int(rtype[q]))
            c = [limit(float(action[q][j]), float(self.cmd[q, j]), (A[j], A[2 + j], A[4 + j]), self.dt) for j in range(2)]
            self.cmd[q] = c
            u[q] = c
            if (A[6:10] != 0.0).any():
                q0, q1 = c[0] * c[0], c[1] * c[1]
                s0, s1 = math.sqrt(A[6] * q0 + A[7] * q1), math.sqrt(A[8] * q0 + A[9] * q1)
                e = q // K if scene is None else int(scene[q // K])
                key = noise_key(self.seed, TAG_MOTION, e, q % K, int(steps[q]))
                u[q] = (c[0] + s0 * normal(key, 0), c[1] + s1 * normal(key, 1))
        return u


def lidar_noise(ranges, hit, K, seed, range_std, range_min, range_max, n=0, envs=None):
    """The noisy float64 ranges of an oracle scan (ranges (N, R) float64 before the float cast, hit (N, R)): a hit gets
    clamp(t + range_std z, range_min, range_max) with z draw i of its robot's lidar stream at step n; ``envs`` the environment
    (scene) of each row's environment (default the row's own, q // K)."""
    out = np.array(ranges, np.float64)
    steps = np.broadcast_to(np.asarray(n, np.int64), (len(out),))
    for q in range(len(out)):
        e = q // K if envs is None else int(envs[q // K])
        idx = np.flatnonzero(np.asarray(hit[q]) >= 0)
        if not len(idx):
            continue
        key = noise_key(seed, TAG_LIDAR, e, q % K, int(steps[q]))
        for i in idx:
            r = float(out[q, i]) + range_std * normal(key, int(i))
            out[q, i] = min(max(r, range_min), range_max)
    return out
