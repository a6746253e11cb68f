"""Continuous episodes on the CPU: a numpy restatement of world_advance_kernel (csrc/world_episode_kernel.cuh) -- the end test and the
slot assignment -- fed per-scene flags and clearances by step of the scene's own episode."""
import numpy as np


class EpisodeOracle:
    """S scenes of K robots through ``slots`` slots, ``max_steps`` steps at most per episode.  ``advance(flags)`` is one
    nb_world_step: ``flags(s, t)`` gives scene s's (collided, arrived, clearance) (K,) arrays after step t of its episode."""

    def __init__(self, S: int, slots: int, K: int, max_steps: int):
        self.S, self.slots, self.K, self.max_steps = S, slots, K, max_steps
        self.scene_of = np.arange(slots, dtype=np.int32)
        self.live = np.ones(slots, np.int32)
        self.reset = np.ones(slots, np.int32)
        self.t = np.zeros(slots, np.int32)
        self.next, self.finished = slots, 0
        self.collided = np.zeros(S * K, np.int32)
        self.arrived = np.zeros(S * K, np.int32)
        self.arrive_step = np.full(S * K, -1, np.int32)
        self.min_clearance = np.full(S * K, np.inf, np.float32)
        self.end_step = np.zeros(S, np.int32)
        self.reason = np.zeros(S, np.int32)
        self.slot = np.full(S, -1, np.int32)
        self.slot[:slots] = np.arange(slots)

    def advance(self, flags):
        K = self.K
        ended = []
        for b in range(self.slots):
            self.reset[b] = 0
            if not self.live[b]:
                continue
            s = int(self.scene_of[b])
            self.t[b] += 1
            t = int(self.t[b])
            col, arr, clear = (np.asarray(a) for a in flags(s, t))
            rows = slice(s * K, (s + 1) * K)
            first = (arr != 0) & (self.arrive_step[rows] < 0)
            self.arrive_step[rows] = np.where(first, t, self.arrive_step[rows])
            self.min_clearance[rows] = np.minimum(self.min_clearance[rows], np.asarray(clear, np.float32))
            done = bool(((col != 0) | (arr != 0)).all())
            if done or t == self.max_steps:
                self.collided[rows], self.arrived[rows] = col, arr
                self.end_step[s], self.reason[s] = t, 1 if done else 2
                ended.append(b)
        for r, b in enumerate(ended):  # ascending slots take ascending scenes
            s = self.next + r
            if s < self.S:
                self.scene_of[b], self.t[b], self.slot[s], self.reset[b] = s, 0, b, 1
            else:
                self.live[b] = 0
        self.next += len(ended)
        self.finished += len(ended)
        return len(ended)

    def run(self, flags, limit: int = 1 << 20):
        """advance until every scene has finished; returns the trace of scene_of before each step (steps, slots)."""
        trace = []
        while self.finished < self.S and len(trace) < limit:
            trace.append(self.scene_of.copy())
            self.advance(flags)
        return np.asarray(trace)
