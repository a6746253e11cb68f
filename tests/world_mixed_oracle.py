"""Float64 restatement of a mixed fleet in the batched world (nb_world_set_fleet_ex), TEST INFRASTRUCTURE ONLY.

``MixedOracleWorld`` is ``oracle.world.OracleWorld`` with robot types: ``types`` are robot types 1..T as dicts of kinematics,
wheelbase and robot_vertices (n, 2) (type 0 is the config's robot) and ``robot_type`` (B K) gives each robot's type.  It performs the
same operations in the same order as the kernels, per robot type: a robot integrates with its type's motion model, its body (what
the other robots' beams cross, what its clearances are taken from) is its type's polygon, and a reactive obstacle sees it as a
circle of its type's circumradius moving with its type's velocity model.  The lidar is shared by every type.  Everything else
(scan, obstacle clearances, reactive obstacles' choice) is OracleWorld's, unchanged; with every robot type 0 this is OracleWorld.
"""
import math

import numpy as np

from oracle.world import OracleWorld, clearance_robot_pairs, integrate, move_obstacle, robot_polygon, robot_velocity


class MixedOracleWorld(OracleWorld):
    def __init__(self, cfg: dict, packed, behaviors=None, seed: int = 0, *, fleet=None, K: int = 1, types=(), robot_type=None):
        super().__init__(cfg, packed, behaviors, seed, fleet=fleet, K=K)
        # the type table: (kinematics, wheelbase, vertices (n, 2), circumradius about the state point)
        self.types = [(cfg["kinematics"], cfg.get("wheelbase"), self.rv, self.robot_r)]
        for t in types:
            tv = np.asarray(t["robot_vertices"], np.float64)
            self.types.append((t["kinematics"], t.get("wheelbase"), tv, max(math.sqrt(x * x + y * y) for x, y in tv)))
        self.rtype = np.zeros(self.N, np.int64) if robot_type is None else np.asarray(robot_type, np.int64).reshape(self.N)

    def type_of(self, n):
        """(kinematics, wheelbase, vertices, circumradius) of robot n's type."""
        return self.types[self.rtype[n]]

    def bodies(self, b):
        return [robot_polygon(self.states[b * self.K + j], self.type_of(b * self.K + j)[2]) for j in range(self.K)]

    def robot_rows(self, b, action):
        """The neighbour rows (x, y, vx, vy, r) of the environment's robots, each with its type's velocity model and circumradius."""
        rows = []
        for n in range(b * self.K, (b + 1) * self.K):
            kin, _, _, r = self.type_of(n)
            v = (0.0, 0.0) if self.collided[n] else robot_velocity(kin, action[n], float(self.states[n, 2]))
            rows.append((float(self.states[n, 0]), float(self.states[n, 1]), v[0], v[1], r))
        return rows

    def robot_clearances(self, bodies):
        """(N,) each robot's smallest clearance to the other robots of its environment (inf with K = 1) from the world vertices of
        every robot (a list of N bodies): clearance_robot_pairs over the pairs of each (vertex count, vertex count) class, which
        takes polygons of different vertex counts on its two sides."""
        K, out = self.K, np.full(self.N, np.inf)
        if K == 1:
            return out
        b, i, j = (a.reshape(-1) for a in np.nonzero(np.broadcast_to(~np.eye(K, dtype=bool), (self.B, K, K))))
        ni, nj = b * K + i, b * K + j
        nv = np.array([len(p) for p in bodies])
        for p, q in sorted(set(zip(nv[ni].tolist(), nv[nj].tolist()))):
            sel = (nv[ni] == p) & (nv[nj] == q)
            P = np.asarray([bodies[n] for n in ni[sel]], np.float64)
            Q = np.asarray([bodies[n] for n in nj[sel]], np.float64)
            np.minimum.at(out, ni[sel], clearance_robot_pairs(P, Q))
        return out

    def step(self, action, rvo=True):
        """OracleWorld.step with each robot's own type: action (N,2) -> (collided, arrived, clearance (N,) float64)."""
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
        for n in range(self.N):
            if clear[n] <= 0.0:
                self.collided[n] = 1
            self.fvel[n] = (0.0, 0.0) if self.collided[n] else vel[n]
        return self.collided.copy(), self.arrived.copy(), clear
