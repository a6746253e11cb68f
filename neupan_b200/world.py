"""Batched 2-D world on the device: lidar scans, moving obstacles and collisions for closed-loop runs of B planners.

The reference evaluates its planner in IR-SIM, one robot at a time in host Python (example/run_exp.py:27-56):
``env.get_robot_state()`` -> ``env.get_lidar_scan()`` -> ``planner(...)`` -> ``env.step(action)`` -> ``env.done()``.
``WorldBatch`` is that loop's world for B environments at once (``nb_world_*``, csrc/world_kernel.cuh), so that a
``PlannerBatch`` runs closed loop without its state ever leaving the GPU; ``rollout`` is the loop itself.

A scene (one environment) is a dict with the sections of an ``env.yaml``:

    obstacles       list of dicts: {"center": (x, y), "radius": r} (circle), {"center": (x, y), "vertices": [[dx, dy], ...]}
                    (convex polygon, 3..8 vertices relative to the centre) or {"center": (x, y), "outline": [[dx, dy], ...]} (any
                    simple polygon, convex or not, either orientation, 3..16 vertices relative to the centre), each with an
                    optional "velocity": (vx, vy) in the world frame (constant unless the obstacle has a behaviour; default
                    still; polygons do not rotate) and an optional "behavior" (below).  At most 256 obstacles and 2048 polygon
                    edges (convex and outline together) per environment.
    bounds          (xmin, ymin, xmax, ymax): a moving obstacle whose centre leaves this rectangle is mirrored back into it and
                    that velocity component is reversed
    start           (x, y, theta) of the robot
    goal            (x, y); goal_threshold: the robot has arrived when it is closer than this to the goal
    path            optional (n, 4) rows [x, y, theta, gear]: an initial path for the planner (the scene builders add one)
    robots          in place of start / goal / goal_threshold / path: a list of K (1..16) dicts with those four keys, the robots of
                    the environment (every scene of a batch has the same K)

An obstacle's "behavior" is {"name": "constant"} (the default) or {"name": "rvo", "vxmax", "vymax", ...} (keys and defaults in
``RVO_DEFAULTS``): a reactive obstacle that heads for a goal at ``speed`` and steers around the other obstacles and the robot with a
reciprocal velocity obstacle over a grid of candidate velocities, before every step moves anything; with ``wander`` it draws a new
goal uniformly in its rectangle on arrival (``goal_threshold``), without it it parks.  This is this project's reading of IR-SIM's
``rvo`` behaviour (IR-SIM is not a dependency), stated in full in csrc/world_rvo_kernel.cuh.  Stated differences from IR-SIM: all
velocities of a step are chosen from the states at its start (IR-SIM updates its objects one after another), obstacles are
holonomic (IR-SIM turns its diff obstacles), every neighbour is a circle (a polygon's circumradius about its centre, the robot's about
its state point), and the candidates are lo + k grid (np.arange can differ in the last bit).  Goals are drawn from counter-based
SplitMix64 streams keyed by (seed, environment, obstacle index within it, draw number), so a run is reproducible from its seed.

Several robots (``robots``, nb_world_set_fleet; this project's reading of an IR-SIM world whose ``robot:`` section is a list): all
share the planner's robot polygon, kinematics and lidar.  Robot k of environment b is row n = b K + k of every per-robot tensor, so
``states``, ``scan``, ``step`` and ``flags`` have N = B K rows and a ``PlannerBatch`` of N planners drives them.  A robot's lidar also
sees the bodies of the other robots of its environment (never its own); a beam that hits robot j reports index O_b + j (after the
O_b obstacles, so an obstacle wins a tie) and that robot's world-frame velocity from the action it integrated in the last step
(translation only; 0 before the first step and once it has collided).  A step is Jacobi: every robot integrates from the state at
the start of the step, then each robot's clearance is the minimum over the obstacles and the other robots (convex-convex, symmetric
bit for bit, so two robots that touch collide in the same step).  A collided robot is frozen and stays in the scene with velocity 0;
an arrived robot stays in the scene.  Reactive obstacles take every robot of their environment as a neighbour.

There is no CPU implementation here: the CUDA library is the product (oracle/world.py restates it for the tests).
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from . import _lib

ENV_COLS = 10  # xmin, ymin, xmax, ymax, start x, y, theta, goal x, y, goal threshold
ROBOT_COLS = 6  # start x, y, theta, goal x, y, goal threshold
MAX_ROBOTS = 16
BEH_COLS = 13  # kind, vxmax, vymax, acce, factor, speed, wander, goal x, y, goal threshold, neighbor range, grid, min speed
# the keys of an "rvo" behaviour besides vxmax and vymax (required); speed None: min(vxmax, vymax); goal None: drawn
RVO_DEFAULTS = dict(acce=1.0, factor=1.0, speed=None, wander=False, goal=None, goal_threshold=0.3, neighbor_range=10.0, grid=0.05,
                    min_speed=0.3)


def make_config(robot, lidar: dict, step_time: float, max_envs: int, device: int = 0) -> _lib.WorldConfig:
    """struct nb_world_config from the planner's robot (its ``vertices`` (2, n), ``kinematics`` and ``L``) and a lidar dict with
    ``angle_min``, ``angle_max``, ``range_max``, ``number`` (R) and optionally ``scan_offset`` (sensor pose in the robot frame)."""
    verts = np.asarray(robot.vertices, dtype=np.float64)
    if verts.ndim != 2 or verts.shape[0] != 2 or verts.shape[1] > 8:
        raise ValueError("robot.vertices must be (2, n) with n <= 8")
    rv = np.zeros(16)
    rv[:2 * verts.shape[1]] = verts.T.reshape(-1)
    return _lib.WorldConfig(kinematics=_lib.NB_KIN[robot.kinematics], num_beams=int(lidar["number"]), max_envs=int(max_envs), device=int(device),
                            robot_num_vertices=verts.shape[1], step_time=float(step_time), wheelbase=float(robot.L or 0.0),
                            angle_min=float(lidar["angle_min"]), angle_max=float(lidar["angle_max"]), range_max=float(lidar["range_max"]),
                            scan_offset=(C.c_double * 3)(*[float(v) for v in lidar.get("scan_offset", (0.0, 0.0, 0.0))]),
                            robot_vertices=(C.c_double * 16)(*rv))


def pack_scenes_ex(scenes):
    """Scenes -> the ragged host arrays of nb_world_set_scenes_ex: obs_begin (B+1) int32, obstacles (O,5) float64 rows
    [cx, cy, vx, vy, radius], vert_begin (O+1) int32, vertices (V,2) float64, envs (B,10) float64, kinds (O) int32
    (0: circle or convex polygon, 1: outline)."""
    obs_begin, rows, vert_begin, verts, envs, kinds = [0], [], [0], [], [], []
    for sc in scenes:
        for ob in sc["obstacles"]:
            vel = ob.get("velocity", (0.0, 0.0))
            if "vertices" in ob and "outline" in ob:
                raise ValueError("an obstacle has either 'vertices' (convex) or 'outline', not both")
            shape = "vertices" if "vertices" in ob else ("outline" if "outline" in ob else None)
            if shape:
                v = np.asarray(ob[shape], dtype=np.float64).reshape(-1, 2)
                verts.append(v)
                vert_begin.append(vert_begin[-1] + v.shape[0])
                rows.append((*ob["center"], *vel, 0.0))
            else:
                vert_begin.append(vert_begin[-1])
                rows.append((*ob["center"], *vel, ob["radius"]))
            kinds.append(1 if shape == "outline" else 0)
        obs_begin.append(len(rows))
        first = sc["robots"][0] if "robots" in sc else sc  # a fleet's env row carries its first robot (unused once the fleet is set)
        envs.append((*sc["bounds"], *first["start"], *first["goal"], first["goal_threshold"]))
    return (np.asarray(obs_begin, np.int32), np.ascontiguousarray(np.asarray(rows, np.float64).reshape(-1, 5)),
            np.asarray(vert_begin, np.int32), np.ascontiguousarray(np.vstack(verts) if verts else np.zeros((0, 2))),
            np.ascontiguousarray(np.asarray(envs, np.float64).reshape(-1, ENV_COLS)), np.asarray(kinds, np.int32))


def pack_scenes(scenes):
    """Scenes of circles and convex polygons -> the ragged host arrays of nb_world_set_scenes: obs_begin (B+1) int32, obstacles
    (O,5) float64 rows [cx, cy, vx, vy, radius], vert_begin (O+1) int32, vertices (V,2) float64, envs (B,10) float64.  Scenes with
    outlines need the kinds of pack_scenes_ex."""
    packed = pack_scenes_ex(scenes)
    if packed[5].any():
        raise ValueError("these scenes have outlines: use pack_scenes_ex (nb_world_set_scenes_ex)")
    return packed[:5]


def fleet_size(scenes) -> int:
    """K: the number of robots of every scene (1 for scenes without ``robots``); raises unless all scenes agree."""
    ks = {len(sc["robots"]) if "robots" in sc else 1 for sc in scenes}
    if len(ks) != 1:
        raise ValueError(f"every scene of a batch needs the same number of robots (got {sorted(ks)})")
    K = ks.pop()
    if not 1 <= K <= MAX_ROBOTS:
        raise ValueError(f"a scene has {K} robots (1..{MAX_ROBOTS})")
    return K


def pack_fleet(scenes) -> np.ndarray:
    """Scenes -> the (B K, 6) float64 rows of nb_world_set_fleet [start x, y, theta, goal x, y, goal_threshold], robot k of
    environment b at row b K + k (a scene without ``robots`` is one robot)."""
    fleet_size(scenes)
    rows = []
    for sc in scenes:
        for rb in (sc["robots"] if "robots" in sc else [sc]):
            rows.append((*rb["start"], *rb["goal"], rb["goal_threshold"]))
    return np.ascontiguousarray(np.asarray(rows, np.float64).reshape(-1, ROBOT_COLS))


def scene_paths(scenes) -> list:
    """The initial paths of every robot in row order (N = B K): the argument of PlannerBatch.set_initial_paths."""
    return [rb["path"] for sc in scenes for rb in (sc["robots"] if "robots" in sc else [sc])]


def pack_behaviors(scenes) -> np.ndarray:
    """Scenes -> the (O, 13) float64 rows of nb_world_set_behaviors, in pack_scenes_ex's obstacle order: [kind (0 constant, 1 rvo),
    vxmax, vymax, acce, factor, speed, wander, goal x, goal y (NaN: drawn), goal_threshold, neighbor_range, grid, min_speed]."""
    rows = []
    for sc in scenes:
        for ob in sc["obstacles"]:
            beh = dict(ob.get("behavior") or {"name": "constant"})
            name = beh.pop("name", None)
            if name == "constant" and not beh:
                rows.append(np.zeros(BEH_COLS))
                continue
            if name != "rvo":
                raise ValueError(f"unknown obstacle behaviour {ob.get('behavior')!r} (\"constant\" or \"rvo\")")
            unknown = set(beh) - set(RVO_DEFAULTS) - {"vxmax", "vymax"}
            if unknown or "vxmax" not in beh or "vymax" not in beh:
                raise ValueError(f"an rvo behaviour needs vxmax and vymax and takes {sorted(RVO_DEFAULTS)} (got {sorted(beh)})")
            p = dict(RVO_DEFAULTS, **beh)
            vxmax, vymax = float(p["vxmax"]), float(p["vymax"])
            speed = min(vxmax, vymax) if p["speed"] is None else float(p["speed"])
            goal = (math.nan, math.nan) if p["goal"] is None else tuple(float(v) for v in p["goal"])
            rows.append(np.array([1.0, vxmax, vymax, p["acce"], p["factor"], speed, 1.0 if p["wander"] else 0.0, *goal,
                                  p["goal_threshold"], p["neighbor_range"], p["grid"], p["min_speed"]], np.float64))
    return np.ascontiguousarray(np.asarray(rows, np.float64).reshape(-1, BEH_COLS))


def _host_ptrs(packed):
    return [C.c_void_p(a.ctypes.data) for a in packed]


class WorldBatch:
    """B environments of one robot type and one lidar, K robots each (``K``, set by the scenes; N = B K).  ``lidar``: angle_min,
    angle_max, range_min, range_max, number (R), optional scan_offset.  ``scan`` / ``step`` enqueue on the current stream and never
    synchronise the host."""

    def __init__(self, num_envs: int, robot, lidar: dict, step_time: float, device=None):
        if not torch.cuda.is_available():
            raise RuntimeError("neupan_b200.WorldBatch needs a CUDA device (no CPU fallback)")
        self.B, self.dt, self.R = int(num_envs), float(step_time), int(lidar["number"])
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.scan_offset = tuple(float(v) for v in lidar.get("scan_offset", (0.0, 0.0, 0.0)))
        self.scan_dict = dict(angle_min=float(lidar["angle_min"]), angle_max=float(lidar["angle_max"]),
                              range_min=float(lidar.get("range_min", 0.0)), range_max=float(lidar["range_max"]))
        self.config = make_config(robot, lidar, step_time, self.B, self.device.index or 0)
        self._handle = C.c_void_p()
        _lib.check(_lib.load().nb_world_create(C.byref(self.config), C.byref(self._handle)))
        self.O = 0
        self.K, self.N = 1, self.B

    def close(self):
        if getattr(self, "_handle", None):
            _lib.load().nb_world_destroy(self._handle)
            self._handle = None

    __del__ = close

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def set_scenes(self, scenes, seed: int = 0):
        """Uploads B scenes, puts every robot at its start and clears the flags (env.reset).  When an obstacle has a behaviour,
        also sets the behaviours (nb_world_set_behaviors); ``seed`` keys the goal draws of reactive obstacles.  Scenes with K > 1
        ``robots`` also set the fleet (nb_world_set_fleet); K = 1 runs as the single-robot world."""
        if len(scenes) != self.B:
            raise ValueError(f"expected {self.B} scenes, got {len(scenes)}")
        K = fleet_size(scenes)
        packed = pack_scenes_ex(scenes)
        fleet = pack_fleet(scenes) if K > 1 else None
        beh = pack_behaviors(scenes) if any("behavior" in ob for sc in scenes for ob in sc["obstacles"]) else None
        with torch.cuda.device(self.device):
            lib = _lib.load()
            if fleet is not None:  # refuse before anything is uploaded
                _lib.check(lib.nb_world_check_fleet(C.byref(self.config), self.B, K, C.c_void_p(fleet.ctypes.data)))
            _lib.check(lib.nb_world_set_scenes_ex(self._handle, self.B, *_host_ptrs(packed)))
            self.O, self.K, self.N = int(packed[0][-1]), 1, self.B
            if beh is not None:
                _lib.check(lib.nb_world_set_behaviors(self._handle, self.B, C.c_void_p(beh.ctypes.data), C.c_uint64(int(seed))))
            if fleet is not None:
                _lib.check(lib.nb_world_set_fleet(self._handle, self.B, K, C.c_void_p(fleet.ctypes.data)))
                self.K, self.N = K, self.B * K

    def goals(self):
        """(goals (O,2) float64, draws (O,) int32) on the device: every obstacle's current goal and the number of goals drawn for it
        so far (zeros for constant-velocity obstacles).  Needs scenes with behaviours."""
        g = torch.empty((self.O, 2), dtype=torch.float64, device=self.device)
        d = torch.empty(self.O, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().nb_world_read_behaviors(self._handle, self.B, C.c_void_p(g.data_ptr()), C.c_void_p(d.data_ptr()), self._stream()))
        return g, d

    def _read(self, states=None, obstacles=None, collided=None, arrived=None):
        p = lambda t: C.c_void_p(0 if t is None else t.data_ptr())
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().nb_world_read_state(self._handle, self.N, p(states), p(obstacles), p(collided), p(arrived), self._stream()))

    @property
    def states(self) -> torch.Tensor:
        """(N,3) float64 [x, y, theta] on the device (env.get_robot_state for every robot): a copy, enqueued on the current stream."""
        s = torch.empty((self.N, 3), dtype=torch.float64, device=self.device)
        self._read(states=s)
        return s

    def obstacles(self) -> torch.Tensor:
        """(O,5) float64 rows [cx, cy, vx, vy, radius] with the current centres and velocities, environments back to back."""
        o = torch.empty((self.O, 5), dtype=torch.float64, device=self.device)
        self._read(obstacles=o)
        return o

    def flags(self):
        """(collided, arrived) (N,) int32, sticky since set_scenes."""
        c, a = (torch.empty(self.N, dtype=torch.int32, device=self.device) for _ in range(2))
        self._read(collided=c, arrived=a)
        return c, a

    def scan(self, hit: bool = False):
        """env.get_lidar_scan() for every robot: (ranges (N,R) f32, velocity (N,2,R) f32, scan dict) -- the arguments of
        PlannerBatch.forward(states, ranges, scan, scan_offset=world.scan_offset, scan_velocity=velocity).  With ``hit``, also the
        index of the object each beam hit within its environment (obstacles, then robot j as O_b + j), -1 on a miss (N,R) int32.  Passing ``velocity`` selects
        scan_to_point_velocity, which applies the sensor offset inversely (neupan.py:271-273): with a non-zero ``scan_offset`` its
        points do not land on the obstacles (the reference's behaviour); without velocities, or at a zero offset, they do."""
        ranges = torch.empty((self.N, self.R), dtype=torch.float32, device=self.device)
        vel = torch.empty((self.N, 2, self.R), dtype=torch.float32, device=self.device)
        hits = torch.empty((self.N, self.R), dtype=torch.int32, device=self.device) if hit else None
        p = lambda t: C.c_void_p(0 if t is None else t.data_ptr())
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().nb_world_scan(self._handle, self.N, p(ranges), p(vel), p(hits), self._stream()))
        return (ranges, vel, dict(self.scan_dict), hits) if hit else (ranges, vel, dict(self.scan_dict))

    def step(self, action):
        """env.step(action) + env.done(): action (N,2) [v, omega] (diff), [v, steering] (acker) or [vx, vy] (omni).
        Returns (collided (N,) int32, arrived (N,) int32, clearance (N,) f32) on the device."""
        action = torch.as_tensor(action).reshape(self.N, 2).to(device=self.device, dtype=torch.float32).contiguous()
        col, arr = (torch.empty(self.N, dtype=torch.int32, device=self.device) for _ in range(2))
        clear = torch.empty(self.N, dtype=torch.float32, device=self.device)
        p = lambda t: C.c_void_p(t.data_ptr())
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().nb_world_step(self._handle, self.N, p(action), p(col), p(arr), p(clear), self._stream()))
        return col, arr, clear


def rollout(planner, world: WorldBatch, steps: int, blind: bool = False, velocities: bool = True):
    """The loop of example/run_exp.py for the world's N robots: scan -> planner.forward -> step, ``steps`` times, all on the device
    and without a host synchronisation of its own.  ``blind``: the planner gets all-range_max scans (it sees nothing) -- the
    baseline that shows what the scans are worth.  ``velocities=False``: the planner gets the scans without their per-beam
    velocities (scan_to_point instead of scan_to_point_velocity) -- what the point velocities are worth.  Returns per-robot
    collided, arrived (bool), steps_to_arrive (int32, -1 = not arrived) and min_clearance (float32, the smallest clearance after
    any step)."""
    B, dev = world.N, world.device
    steps_to_arrive = torch.full((B,), -1, dtype=torch.int32, device=dev)
    min_clear = torch.full((B,), math.inf, dtype=torch.float32, device=dev)
    if blind:
        blind_ranges = torch.full((B, world.R), world.scan_dict["range_max"], dtype=torch.float32, device=dev)
        blind_vel = torch.zeros((B, 2, world.R), dtype=torch.float32, device=dev)
        blind_scan = dict(world.scan_dict)
    for k in range(steps):
        ranges, vel, scan = (blind_ranges, blind_vel, blind_scan) if blind else world.scan()
        action, _ = planner.forward(world.states, ranges, scan, scan_offset=world.scan_offset, scan_velocity=vel if velocities else None)
        _, arrived, clearance = world.step(action)
        steps_to_arrive = torch.where((arrived != 0) & (steps_to_arrive < 0), k + 1, steps_to_arrive)
        min_clear = torch.minimum(min_clear, clearance)
    collided, arrived = world.flags()
    return dict(collided=collided.bool(), arrived=arrived.bool(), steps_to_arrive=steps_to_arrive, min_clearance=min_clear)


# ---- seeded scenes after the reference's examples -------------------------------------------------------------------------

def _rng(seed: int, b: int) -> np.random.Generator:
    """Environment b's own child stream (as synth.make_inputs): any sub-range of environments reproduces the same scenes."""
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed, spawn_key=(b,))))


def rectangle(length: float, width: float, theta: float = 0.0) -> np.ndarray:
    """Vertices (4,2) of a length x width rectangle centred on its centre and turned by theta (IR-SIM's 'rectangle' shape)."""
    c, s = math.cos(theta), math.sin(theta)
    corners = np.array([[-length / 2, -width / 2], [length / 2, -width / 2], [length / 2, width / 2], [-length / 2, width / 2]])
    return corners @ np.array([[c, s], [-s, c]])


def line_path(start, goal, spacing: float = 0.1) -> np.ndarray:
    """(n,4) rows [x, y, theta, gear = 1] along the segment start -> goal (the 'line' curve of two waypoints)."""
    d = math.hypot(goal[0] - start[0], goal[1] - start[1])
    n = max(2, int(math.ceil(d / spacing)) + 1)
    s = np.linspace(0.0, 1.0, n)
    th = math.atan2(goal[1] - start[1], goal[0] - start[0])
    return np.stack([start[0] + s * (goal[0] - start[0]), start[1] + s * (goal[1] - start[1]), np.full(n, th), np.ones(n)], 1)


def corridor(num_envs: int, seed: int = 0, circles: int = 4):
    """example/corridor/diff/env.yaml: a 70 x 23 m world at offset (-3, 10), two 70 x 2 m walls centred at (30, 25) and (30, 15)
    (a corridor 8 m wide around y = 20), goal threshold 0.3; the planner's path runs from (0, 20) to (60, 20)
    (example/corridor/diff/planner.yaml).  Instead of the example's four turned blocks, ``circles`` static circles of radius
    0.4..0.8 m stand in the corridor (x in 10..50 m, y in 17.5..22.5 m); the robot starts at (0, 20 +- 1, 0)."""
    scenes = []
    for b in range(num_envs):
        rng = _rng(seed, b)
        start = (0.0, 20.0 + rng.uniform(-1.0, 1.0), 0.0)
        goal = (60.0, 20.0)
        obs = [dict(center=(30.0, 25.0), vertices=rectangle(70.0, 2.0)), dict(center=(30.0, 15.0), vertices=rectangle(70.0, 2.0))]
        for _ in range(circles):
            obs.append(dict(center=(rng.uniform(10.0, 50.0), rng.uniform(17.5, 22.5)), radius=rng.uniform(0.4, 0.8)))
        scenes.append(dict(obstacles=obs, bounds=(-3.0, 10.0, 67.0, 33.0), start=start, goal=goal, goal_threshold=0.3,
                           path=line_path(start, goal)))
    return scenes


# the obstacles' behaviour in example/dyna_obs and example/dyna_non_obs: {name: 'rvo', wander: True, vxmax: 0.5, vymax: 0.5}, with
# goal threshold 0.3 for the examples' arrive_mode: position; the other keys at RVO_DEFAULTS
EXAMPLE_RVO = dict(name="rvo", vxmax=0.5, vymax=0.5, wander=True, goal_threshold=0.3)


def _apply_behavior(obs, behavior: str):
    """behavior "constant": the obstacles as drawn; "rvo": the same obstacles at rest with EXAMPLE_RVO (goals drawn on the device)."""
    if behavior == "constant":
        return obs
    if behavior != "rvo":
        raise ValueError(f"behavior must be 'constant' or 'rvo' (got {behavior!r})")
    return [dict(ob, velocity=(0.0, 0.0), behavior=dict(EXAMPLE_RVO)) for ob in obs]


def dyna_obs(num_envs: int, seed: int = 0, count: int = 20, behavior: str = "constant"):
    """example/dyna_obs/diff/env.yaml: ``count`` (20) circles of radius 0.4..1.0 m placed at random in the box [10, 40]^2, goal
    threshold 0.4.  ``behavior="constant"``: each moves at a constant speed of at most 0.5 m/s in a random direction and bounces
    inside that box.  ``behavior="rvo"``: the example's reactive obstacles (EXAMPLE_RVO: vxmax = vymax = 0.5, wander, goal threshold
    0.3), starting at rest at the same centres.  The robot crosses the box: it starts at (6, y0) facing the goal (44, y1), y0, y1 in
    15..35 m, on a straight path."""
    scenes = []
    for b in range(num_envs):
        rng = _rng(seed, b)
        y0, y1 = rng.uniform(15.0, 35.0, 2)
        start = (6.0, y0, math.atan2(y1 - y0, 38.0))
        goal = (44.0, y1)
        c = rng.uniform(10.0, 40.0, (count, 2))
        r = rng.uniform(0.4, 1.0, count)
        speed, heading = rng.uniform(0.0, 0.5, count), rng.uniform(-math.pi, math.pi, count)
        obs = [dict(center=(c[i, 0], c[i, 1]), radius=r[i], velocity=(speed[i] * math.cos(heading[i]), speed[i] * math.sin(heading[i])))
               for i in range(count)]
        obs = _apply_behavior(obs, behavior)
        scenes.append(dict(obstacles=obs, bounds=(10.0, 10.0, 40.0, 40.0), start=start, goal=goal, goal_threshold=0.4,
                           path=line_path(start, goal)))
    return scenes


def random_outline(rng: np.random.Generator, avg_radius: float, irregularity: float, spikeyness: float, n_vertices: int) -> np.ndarray:
    """Vertices (n,2) of a random star-shaped polygon around the centre (0, 0): this project's reading of IR-SIM's `random_shape`
    polygons (the well-known random-polygon recipe; IR-SIM itself is not a dependency, so its polygons are not compared).

    The angular steps are drawn from U(2 pi / n (1 - irregularity), 2 pi / n (1 + irregularity)) and normalised to sum to 2 pi,
    from a random first angle; the radii from N(avg_radius, spikeyness * avg_radius), clipped to [0.1, 2] * avg_radius so that no
    vertex collapses onto the centre.  Steps are drawn again while one of them reaches pi: with every step in (0, pi) the centre
    sees the vertices in strictly increasing directions, each edge stays in its own sector, and the polygon is simple (usually not
    convex)."""
    n = int(n_vertices)
    mean = 2.0 * math.pi / n
    while True:
        steps = rng.uniform(mean * (1.0 - irregularity), mean * (1.0 + irregularity), n)
        steps *= 2.0 * math.pi / steps.sum()
        if steps.max() < math.pi and steps.min() > 0.0:
            break
    angles = rng.uniform(0.0, 2.0 * math.pi) + np.concatenate([[0.0], np.cumsum(steps[:-1])])
    r = np.clip(rng.normal(avg_radius, spikeyness * avg_radius, n), 0.1 * avg_radius, 2.0 * avg_radius)
    return np.stack([r * np.cos(angles), r * np.sin(angles)], 1)


def _example_outline(rng, avg_radius: float, irregularity: float) -> np.ndarray:
    """An outline of the reference's `random_shape: true` obstacles: 4..9 vertices and spikeyness U(0, 1) (a stated choice: the
    examples give only the radius and irregularity ranges)."""
    spikeyness, n = rng.uniform(0.0, 1.0), int(rng.integers(4, 10))
    return random_outline(rng, avg_radius, irregularity, spikeyness, n)


def dyna_non_obs(num_envs: int, seed: int = 0, behavior: str = "constant"):
    """example/dyna_non_obs/diff/{env,planner}.yaml: 11 obstacles, each one of the example's four shapes drawn uniformly -- the
    2 x 2 m square, a circle of r = 1.5, a circle of r = 1.0, or an outline of average radius U(0.5, 1.5) and irregularity 0.9 (how
    IR-SIM assigns a 4-entry shape list to 11 obstacles is a stated choice here).  Centres uniform in [5, 45] x [15, 35].
    ``behavior="constant"``: constant velocities (vx, vy) in U(-1, 1)^2, bouncing in that box.  ``behavior="rvo"``: the example's
    reactive obstacles (EXAMPLE_RVO), circles, squares and outlines alike, starting at rest at the same centres.  The robot starts
    at (-1, 25, 0) on the planner's line path to (50, 25), its goal, with threshold 0.4."""
    square = [[-1.0, -1.0], [1.0, -1.0], [1.0, 1.0], [-1.0, 1.0]]
    start, goal = (-1.0, 25.0, 0.0), (50.0, 25.0)
    scenes = []
    for b in range(num_envs):
        rng = _rng(seed, b)
        obs = []
        for _ in range(11):
            shape = int(rng.integers(0, 4))
            ob = dict(center=tuple(rng.uniform((5.0, 15.0), (45.0, 35.0))), velocity=tuple(rng.uniform(-1.0, 1.0, 2)))
            if shape == 0:
                ob["vertices"] = square
            elif shape in (1, 2):
                ob["radius"] = 1.5 if shape == 1 else 1.0
            else:
                ob["outline"] = _example_outline(rng, rng.uniform(0.5, 1.5), 0.9)
            obs.append(ob)
        obs = _apply_behavior(obs, behavior)
        scenes.append(dict(obstacles=obs, bounds=(5.0, 15.0, 45.0, 35.0), start=start, goal=goal, goal_threshold=0.4,
                           path=line_path(start, goal)))
    return scenes


# the first 11 `state` rows of example/non_obs/acker/env.yaml (its list has 12 for 11 obstacles; the repeated (16, 26) is kept)
NON_OBS_CENTRES = ((20.0, 34.0), (31.0, 38.0), (10.0, 20.0), (41.0, 25.0), (18.8, 13.0), (16.0, 26.0), (10.0, 24.0), (15.0, 20.0),
                   (16.0, 26.0), (19.0, 26.0), (11.0, 14.5))


def non_obs(num_envs: int, seed: int = 0):
    """example/non_obs/acker/{env,planner}.yaml: 11 static outlines at the example's positions, average radius U(0.5, 1.0) and
    irregularity U(0.9, 1.0), different in every environment; the world's rectangle (-2, 5, 51, 47).  The robot starts at
    (-1, 25, 0) with goal (50, 25) and threshold 0.3; the example's dubins curve between these two poses is the straight line."""
    start, goal = (-1.0, 25.0, 0.0), (50.0, 25.0)
    scenes = []
    for b in range(num_envs):
        rng = _rng(seed, b)
        obs = [dict(center=c, outline=_example_outline(rng, rng.uniform(0.5, 1.0), rng.uniform(0.9, 1.0))) for c in NON_OBS_CENTRES]
        scenes.append(dict(obstacles=obs, bounds=(-2.0, 5.0, 51.0, 47.0), start=start, goal=goal, goal_threshold=0.3,
                           path=line_path(start, goal)))
    return scenes


def circle_swap(num_envs: int, robots: int = 8, radius: float = 10.0, seed: int = 0, circles: int = 0):
    """The standard multi-robot benchmark: ``robots`` robots evenly spaced on a circle of ``radius`` about (0, 0), each facing its
    antipode, which is its goal (threshold 0.3), on a line path.  Per environment the circle turns by a random angle and every robot
    gets a small jitter (0.1 m in position, 0.05 rad in heading) so that the configuration is not exactly symmetric.  ``circles``
    static circles of radius 0.3..0.6 m stand within radius / 3 of the centre.  Rectangle [-(radius + 3), radius + 3]^2.  At the
    default radius of 10 m, 16 robots of C4's 1.6 x 2.0 m body start about 1.9 m apart.  Seeded per environment (``_rng``)."""
    K = int(robots)
    if not 1 <= K <= MAX_ROBOTS:
        raise ValueError(f"robots must be in 1..{MAX_ROBOTS} (got {K})")
    ext = radius + 3.0
    scenes = []
    for b in range(num_envs):
        rng = _rng(seed, b)
        rot = rng.uniform(0.0, 2.0 * math.pi)
        jit = rng.uniform(-1.0, 1.0, (K, 3)) * np.array([0.1, 0.1, 0.05])
        fleet = []
        for k in range(K):
            a = rot + 2.0 * math.pi * k / K
            sx, sy = radius * math.cos(a) + jit[k, 0], radius * math.sin(a) + jit[k, 1]
            goal = (-radius * math.cos(a), -radius * math.sin(a))
            start = (sx, sy, math.atan2(goal[1] - sy, goal[0] - sx) + jit[k, 2])
            fleet.append(dict(start=start, goal=goal, goal_threshold=0.3, path=line_path(start, goal)))
        obs = []
        for _ in range(circles):
            r, a = rng.uniform(0.0, radius / 3.0), rng.uniform(0.0, 2.0 * math.pi)
            obs.append(dict(center=(r * math.cos(a), r * math.sin(a)), radius=rng.uniform(0.3, 0.6)))
        scenes.append(dict(obstacles=obs, bounds=(-ext, -ext, ext, ext), robots=fleet))
    return scenes
