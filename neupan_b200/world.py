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
    map             optional static occupancy grid {"occupancy": (H, W) bool array, row 0 the lowest y, "origin": (x, y) the
                    lower-left corner of cell (0, 0), "resolution": r the side of a cell in m} (1..8192 cells per side, r >= 0.01):
                    this project's reading of IR-SIM's ``world: obstacle_map:``.  Cells outside the grid are free.  The lidar sees
                    where a beam crosses from a free into an occupied cell (hit index O_b + K, velocity 0), the step takes the exact
                    clearance to the occupied cells within ``map_window`` of each robot (csrc/world_kernel.cuh states the rules).
                    Scenes that share one occupancy array (the same object, origin and resolution) share one copy of it on the
                    device.  By default reactive obstacles do not see the map and moving obstacles pass over it; with
                    ``"blocks_obstacles": True`` the map blocks the scene's obstacles (below).

Obstacles in occupancy maps (``"map": {..., "blocks_obstacles": True}``, nb_world_set_map_contact): a moving obstacle whose move
would make its footprint touch an occupied cell takes instead the x move alone (y velocity reversed), else the y move alone (x
velocity reversed), else stays in place with both reversed -- a bounce, counted per obstacle by ``map_bounces()``.  A reactive
obstacle's wander goal must have a clear footprint and a straight segment to it that keeps more than the obstacle's circumradius from
every occupied cell (at most 16 draws per step, else it waits a step); after a bounce it draws a new goal.  Every moving obstacle of
such a scene must start clear of the map, and its top speed times step_time must be below the map's resolution.  Walls are not RVO
neighbours, obstacles pass through each other unless the scene has obstacle contact (below), and motion is not swept
(csrc/world_kernel.cuh states the rules).

Obstacle contact (a scene's ``"obstacle_contact": True``, nb_world_set_obstacle_contact): the scene's obstacles block each other.
They move one after another in list order, each tested against the others where they stand at that moment (the earlier ones already
moved), which is how IR-SIM moves its objects.  A moving obstacle whose move would make its footprint touch another obstacle (or a map
that blocks obstacles) takes instead the x move alone (y velocity reversed), else the y move alone (x velocity reversed), else stays in
place with both reversed -- an obstacle bounce, counted per obstacle by ``obstacle_bounces()``.  So no moving obstacle ever touches
another obstacle.  Every moving obstacle of such a scene must start clear of the others; static obstacles may overlap each other.
Robots do not block obstacles, motion is not swept (a step longer than the thinner of two footprints can pass through it), and there
is no momentum or elastic response (csrc/world_contact_kernel.cuh states the rules).  The builders ``dyna_obs``, ``dyna_non_obs``,
``maze`` and ``cave`` take ``contact=True`` to place their obstacles clear of each other and set the key.

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

Mixed fleets (nb_world_set_fleet_ex): ``WorldBatch`` takes a sequence of robots, entry i being robot type i (type 0 gives the
config), and a scene robot (or a single-robot scene) may carry ``"type": i`` (default 0), so robots of different shapes and
kinematics share a world, at most 4 types.  Each robot integrates with its type's motion model, its body (what the other robots see
and collide with) is its type's polygon, and reactive obstacles see it with its type's circumradius and velocity model; the lidar is
shared by every type, so scans stay (N, R).  Actions are in each robot's own convention (omni: (vx, vy)).  ``rows_of_type(i)`` gives
the rows of one kind, ``scene_paths(scenes, type=i)`` their paths, and ``MixedPlanner`` drives every kind with its own
``PlannerBatch`` behind one ``forward``, so ``rollout`` runs a mixed world unchanged.  K = 1 is allowed: one robot per environment,
of any type (the same seeded scenes with a diff, an acker and an omni robot side by side).

Continuous episodes (nb_world_set_episodes, ``WorldBatch.set_episodes``, ``run_episodes``): a bank of S scenes runs through B
slots.  When a slot's episode ends (every robot of its scene collided or arrived, or ``max_steps`` steps), the slot takes the next
unstarted scene on the device: the slots that ended, in ascending order, take the next scenes in ascending order.  Once the bank is
exhausted a slot goes idle and its scene is frozen.  Each scene runs once in its own rows, so an episode is bitwise the plain run of
its scene truncated at its end.  The per-scene results are read with ``episodes()``.  Limits: one ``max_steps`` per world, no
differentiable mode, a single GPU, the bank within ``num_envs`` and device memory, a fixed type per robot index.

Actuation limits and noise (``WorldBatch.set_actuation``, ``set_lidar_noise``; nb_world_set_actuation, nb_world_set_lidar_noise):
both off by default, and a world without them runs the kernels it ran before.  This is this project's reading of IR-SIM's
``vel_min`` / ``vel_max`` / ``acce`` and of the ``noise`` switches of its motion model and ``lidar2d``, not a claim of parity.
``set_actuation`` takes one dict per robot type with the keys ``vel_min``, ``vel_max`` (2 values each, default -inf / +inf),
``acce`` (2, default +inf) and ``alpha`` (4, default 0), in the action's own convention: diff (v, omega), acker (v, steering), omni
(vx, vy).  Each robot carries cmd_prev, its last limited command (``commands()``; 0 after set_scenes / set_episodes and when a slot
takes a new scene).  In a step, per component, lo = max(vel_min, cmd_prev - acce dt), hi = min(vel_max, cmd_prev + acce dt),
c = min(max(a, lo), hi) and cmd_prev = c; then s0 = sqrt(alpha0 c0^2 + alpha1 c1^2), s1 = sqrt(alpha2 c0^2 + alpha3 c1^2) and the
robot integrates u = c + (s0 z0, s1 z1) with its type's motion model; the velocity the lidar reports for it is that of u.  Noise comes
after the limits and is not clipped again (IR-SIM's order).  A collided robot stays frozen and its cmd_prev becomes 0.  Reactive
obstacles still see the action as given.  ``set_lidar_noise(range_std, range_min)``: a beam that hits something reports
clamp(t + range_std z, range_min, range_max), computed in FP64 and rounded to float; a miss still reports range_max, and the hit
index and velocity do not change.  z are standard normal draws (Box-Muller from SplitMix64 counter streams, one domain tag for motion
and one for the lidar, apart from the goal draws) keyed by (seed, environment -- the scene in episode mode --, robot within it, the
steps that scene has taken, component or beam), so a run is reproducible from its seeds, environment b's noise does not depend on B,
a scan repeated without a step is the same scan, and an episode stays bitwise the plain run of its scene.  The settings survive
set_scenes and set_episodes.  Refused (ValueError): NaN, vel_min > vel_max, acce <= 0, negative or non-finite alpha, and an acker
type's finite steering limits outside (-pi/2, pi/2).

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
MAX_ROBOT_TYPES = 4
BEH_COLS = 13  # kind, vxmax, vymax, acce, factor, speed, wander, goal x, y, goal threshold, neighbor range, grid, min speed
# the keys of an "rvo" behaviour besides vxmax and vymax (required); speed None: min(vxmax, vymax); goal None: drawn
RVO_DEFAULTS = dict(acce=1.0, factor=1.0, speed=None, wander=False, goal=None, goal_threshold=0.3, neighbor_range=10.0, grid=0.05,
                    min_speed=0.3)
# the keys of a robot type's actuation (WorldBatch.set_actuation) and their defaults: no bound, no rate limit, no motion noise
ACTUATION_DEFAULTS = dict(vel_min=(-math.inf, -math.inf), vel_max=(math.inf, math.inf), acce=(math.inf, math.inf), alpha=(0.0, 0.0, 0.0, 0.0))


def _robot_vertices(robot):
    verts = np.asarray(robot.vertices, dtype=np.float64)
    if verts.ndim != 2 or verts.shape[0] != 2 or verts.shape[1] > 8:
        raise ValueError("robot.vertices must be (2, n) with n <= 8")
    rv = np.zeros(16)
    rv[:2 * verts.shape[1]] = verts.T.reshape(-1)
    return verts, rv


def make_robot_type(robot) -> _lib.WorldRobotType:
    """struct nb_world_robot_type from a robot (its ``vertices`` (2, n), ``kinematics`` and ``L``)."""
    verts, rv = _robot_vertices(robot)
    return _lib.WorldRobotType(kinematics=_lib.NB_KIN[robot.kinematics], num_vertices=verts.shape[1], wheelbase=float(robot.L or 0.0),
                               vertices=(C.c_double * 16)(*rv))


def make_config(robot, lidar: dict, step_time: float, max_envs: int, device: int = 0) -> _lib.WorldConfig:
    """struct nb_world_config from the planner's robot (its ``vertices`` (2, n), ``kinematics`` and ``L``) and a lidar dict with
    ``angle_min``, ``angle_max``, ``range_max``, ``number`` (R) and optionally ``scan_offset`` (sensor pose in the robot frame)."""
    verts, rv = _robot_vertices(robot)
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


def pack_robot_types(scenes) -> np.ndarray:
    """Scenes -> the (B K) int32 robot types of nb_world_set_fleet_ex in pack_fleet's row order (a robot's ``type``, default 0)."""
    fleet_size(scenes)
    return np.ascontiguousarray([int(rb.get("type", 0)) for sc in scenes for rb in (sc["robots"] if "robots" in sc else [sc])], np.int32)


def scene_paths(scenes, type: int = None) -> list:
    """The initial paths of every robot in row order (N = B K): the argument of PlannerBatch.set_initial_paths.  With ``type``,
    only the robots of that type, in row order (the rows of WorldBatch.rows_of_type)."""
    return [rb["path"] for sc in scenes for rb in (sc["robots"] if "robots" in sc else [sc]) if type is None or rb.get("type", 0) == type]


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


def pack_maps(scenes):
    """Scenes -> the host arrays of nb_world_set_maps: maps (P) of struct nb_world_map, bits (words,) uint32 (each map ``height``
    rows of ceil(width / 32) words, bit i mod 32 of word i / 32 being cell (i, j), padding bits 0), env_map (B) int32 (-1: no map).
    A map shared by several scenes (the same occupancy array object, origin and resolution) is stored once."""
    index, structs, chunks, env_map = {}, [], [], []
    for sc in scenes:
        m = sc.get("map")
        if m is None:
            env_map.append(-1)
            continue
        origin, res = tuple(float(v) for v in m["origin"]), float(m["resolution"])
        key = (id(m["occupancy"]), origin, res)
        if key not in index:
            occ = np.asarray(m["occupancy"], bool)
            if occ.ndim != 2:
                raise ValueError(f"a map's occupancy must be an (H, W) array (got shape {occ.shape})")
            H, W = occ.shape
            words = (W + 31) // 32
            padded = np.zeros((H, 32 * words), bool)
            padded[:, :W] = occ
            chunks.append(np.packbits(padded, axis=1, bitorder="little").view("<u4").astype(np.uint32).reshape(-1))
            index[key] = len(structs)
            structs.append(_lib.WorldMap(width=W, height=H, origin=(C.c_double * 2)(*origin), resolution=res))
        env_map.append(index[key])
    maps = (_lib.WorldMap * max(1, len(structs)))(*structs)
    bits = np.ascontiguousarray(np.concatenate(chunks) if chunks else np.zeros(1, np.uint32))
    return maps, bits, np.ascontiguousarray(env_map, np.int32)


def pack_map_contact(scenes) -> np.ndarray:
    """Scenes -> the (B) int32 flags of nb_world_set_map_contact: 1 where the scene's map has ``"blocks_obstacles": True``."""
    return np.ascontiguousarray([1 if (sc.get("map") or {}).get("blocks_obstacles", False) else 0 for sc in scenes], np.int32)


def pack_obstacle_contact(scenes) -> np.ndarray:
    """Scenes -> the (B) int32 flags of nb_world_set_obstacle_contact: 1 where the scene has ``"obstacle_contact": True``."""
    return np.ascontiguousarray([1 if sc.get("obstacle_contact", False) else 0 for sc in scenes], np.int32)


def pack_actuation(limits, robots) -> np.ndarray:
    """(T, 10) float64 rows [vel_min (2), vel_max (2), acce (2), alpha (4)] from one dict per robot type (``robots``: the world's
    robot types, whose kinematics decide the acker check), with the refusals of nb_world_set_actuation as ValueError naming the type."""
    if len(limits) != len(robots):
        raise ValueError(f"{len(limits)} actuation dicts for {len(robots)} robot types")
    rows = []
    for t, (lim, robot) in enumerate(zip(limits, robots)):
        unknown = set(lim) - set(ACTUATION_DEFAULTS)
        if unknown:
            raise ValueError(f"robot type {t}: unknown actuation keys {sorted(unknown)}")
        v = {k: np.asarray(lim.get(k, d), np.float64).reshape(-1) for k, d in ACTUATION_DEFAULTS.items()}
        for k, d in ACTUATION_DEFAULTS.items():
            if v[k].shape != (len(d),):
                raise ValueError(f"robot type {t}: {k} needs {len(d)} values, got {v[k].size}")
            if np.isnan(v[k]).any():
                raise ValueError(f"robot type {t}: {k} = {v[k].tolist()} has a NaN")
        lo, hi = v["vel_min"], v["vel_max"]
        if (lo > hi).any() or (lo == math.inf).any() or (hi == -math.inf).any():
            raise ValueError(f"robot type {t}: vel_min = {lo.tolist()} and vel_max = {hi.tolist()} need vel_min <= vel_max (vel_min < inf, "
                             "vel_max > -inf)")
        if (v["acce"] <= 0.0).any():
            raise ValueError(f"robot type {t}: acce = {v['acce'].tolist()} must be > 0 (inf: no rate limit)")
        if not np.isfinite(v["alpha"]).all() or (v["alpha"] < 0.0).any():
            raise ValueError(f"robot type {t}: alpha = {v['alpha'].tolist()} must be finite and >= 0")
        if robot.kinematics == "acker":
            steer = np.array([lo[1], hi[1]])
            fin = steer[np.isfinite(steer)]
            if (np.abs(fin) >= math.pi / 2).any():
                raise ValueError(f"robot type {t} (acker): steering limits {steer.tolist()} outside (-pi/2, pi/2)")
        rows.append(np.concatenate([lo, hi, v["acce"], v["alpha"]]))
    return np.asarray(rows, np.float64).reshape(len(robots), 10)


def check_lidar_noise(range_std: float, range_min: float, range_max: float):
    """The refusals of nb_world_set_lidar_noise as ValueError: range_std finite and >= 0, range_min in [0, range_max)."""
    if not (math.isfinite(range_std) and range_std >= 0.0):
        raise ValueError(f"range_std = {range_std} must be finite and >= 0")
    if not 0.0 <= range_min < range_max:
        raise ValueError(f"range_min = {range_min} outside [0, range_max = {range_max})")


def _host_ptrs(packed):
    return [C.c_void_p(a.ctypes.data) for a in packed]


class WorldBatch:
    """B environments of one lidar, K robots each (``K``, set by the scenes; N = B K).  ``robot``: the robot, or a sequence of
    robots whose entry i is robot type i (a mixed fleet, at most 4 types; the scenes' robots choose theirs with ``"type"``).
    ``lidar``: angle_min, angle_max, range_min, range_max, number (R), optional scan_offset.  ``scan`` / ``step`` enqueue on the
    current stream and never synchronise the host."""

    def __init__(self, num_envs: int, robot, lidar: dict, step_time: float, device=None):
        robots = list(robot) if isinstance(robot, (list, tuple)) else [robot]
        if not 1 <= len(robots) <= MAX_ROBOT_TYPES:
            raise ValueError(f"1..{MAX_ROBOT_TYPES} robot types (got {len(robots)})")
        robot = robots[0]
        self.robots = robots
        self.types = (_lib.WorldRobotType * max(1, len(robots) - 1))(*[make_robot_type(r) for r in robots[1:]])
        self._rows = None
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
        self._envs, self.S, self.slots = self.B, None, None  # environments on the device; the bank and slots in episode mode

    def close(self):
        if getattr(self, "_handle", None):
            _lib.load().nb_world_destroy(self._handle)
            self._handle = None

    __del__ = close

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def set_scenes(self, scenes, seed: int = 0, map_window: float = 1.0):
        """Uploads B scenes, puts every robot at its start and clears the flags (env.reset).  When an obstacle has a behaviour,
        also sets the behaviours (nb_world_set_behaviors); ``seed`` keys the goal draws of reactive obstacles.  Scenes with K > 1
        ``robots`` also set the fleet (nb_world_set_fleet); K = 1 runs as the single-robot world.  With several robot types the
        fleet goes through nb_world_set_fleet_ex with every robot's ``type`` (any K).  When a scene has a ``map``, also sets the
        maps (nb_world_set_maps, pack_maps) with ``map_window`` (m, in (0, 10]): a robot's map clearance is exact up to it and
        reported as ``map_window`` beyond."""
        if len(scenes) != self.B:
            raise ValueError(f"expected {self.B} scenes, got {len(scenes)}")
        self._upload(scenes, seed, map_window)

    def _upload(self, scenes, seed: int, map_window: float):
        """set_scenes for B = len(scenes) <= num_envs environments (the world leaves episode mode)."""
        B = len(scenes)
        K = fleet_size(scenes)
        packed = pack_scenes_ex(scenes)
        rtype = pack_robot_types(scenes)
        T = len(self.robots) - 1
        if T == 0 and rtype.any():
            raise ValueError(f"a robot has type {int(rtype.max())} but the world has one robot type")
        fleet = pack_fleet(scenes) if K > 1 or T > 0 else None
        beh = pack_behaviors(scenes) if any("behavior" in ob for sc in scenes for ob in sc["obstacles"]) else None
        maps = pack_maps(scenes) if any("map" in sc for sc in scenes) else None
        contact = pack_map_contact(scenes) if maps is not None else None
        if contact is not None and not contact.any():
            contact = None
        ocontact = pack_obstacle_contact(scenes) if any("obstacle_contact" in sc for sc in scenes) else None
        if ocontact is not None and not ocontact.any():
            ocontact = None
        with torch.cuda.device(self.device):
            lib = _lib.load()
            fleet_args = (B, K, C.c_void_p(fleet.ctypes.data)) if fleet is not None else None
            types_args = (T, self.types) if T > 0 else None
            if fleet is not None:  # refuse before anything is uploaded
                if types_args:
                    _lib.check(lib.nb_world_check_fleet_ex(C.byref(self.config), *types_args, *fleet_args, C.c_void_p(rtype.ctypes.data)))
                else:
                    _lib.check(lib.nb_world_check_fleet(C.byref(self.config), *fleet_args))
            if maps is not None:
                rows = pack_fleet(scenes)
                map_args = (len(maps[0]), maps[0], C.c_void_p(maps[1].ctypes.data),
                            C.c_void_p(maps[2].ctypes.data), C.c_double(float(map_window)))
                _lib.check(lib.nb_world_check_maps(C.byref(self.config), T, self.types, B, K, C.c_void_p(rows.ctypes.data),
                                                   C.c_void_p(rtype.ctypes.data), *map_args))
            if contact is not None:
                bptr = C.c_void_p(beh.ctypes.data) if beh is not None else C.c_void_p(0)
                _lib.check(lib.nb_world_check_map_contact(C.byref(self.config), B, *_host_ptrs(packed), bptr, *map_args[:4],
                                                          C.c_void_p(contact.ctypes.data)))
            if ocontact is not None:
                bptr = C.c_void_p(beh.ctypes.data) if beh is not None else C.c_void_p(0)
                _lib.check(lib.nb_world_check_obstacle_contact(C.byref(self.config), B, *_host_ptrs(packed), bptr,
                                                               C.c_void_p(ocontact.ctypes.data)))
            _lib.check(lib.nb_world_set_scenes_ex(self._handle, B, *_host_ptrs(packed)))
            self.O, self.K, self.N = int(packed[0][-1]), 1, B
            self._envs, self.S, self.slots = B, None, None
            self._rows = None
            if beh is not None:
                _lib.check(lib.nb_world_set_behaviors(self._handle, B, C.c_void_p(beh.ctypes.data), C.c_uint64(int(seed))))
            if fleet is not None:
                if types_args:
                    _lib.check(lib.nb_world_set_fleet_ex(self._handle, *types_args, *fleet_args, C.c_void_p(rtype.ctypes.data)))
                else:
                    _lib.check(lib.nb_world_set_fleet(self._handle, *fleet_args))
                self.K, self.N = K, B * K
            if maps is not None:
                _lib.check(lib.nb_world_set_maps(self._handle, *map_args))
            if contact is not None:
                _lib.check(lib.nb_world_set_map_contact(self._handle, B, C.c_void_p(contact.ctypes.data)))
            if ocontact is not None:
                _lib.check(lib.nb_world_set_obstacle_contact(self._handle, B, C.c_void_p(ocontact.ctypes.data)))
        self.map_contact = contact is not None
        self.obstacle_contact = ocontact is not None
        self.robot_types = rtype
        self._rows = [torch.from_numpy(np.flatnonzero(rtype == i)).to(self.device) for i in range(len(self.robots))]

    def rows_of_type(self, i: int) -> torch.Tensor:
        """The rows (int64, on the device, ascending) of the robots of type i, built once by set_scenes."""
        if self._rows is None:
            raise ValueError("no scenes set")
        return self._rows[i]

    def goals(self):
        """(goals (O,2) float64, draws (O,) int32) on the device: every obstacle's current goal and the number of goals drawn for it
        so far (zeros for constant-velocity obstacles).  Needs scenes with behaviours."""
        g = torch.empty((self.O, 2), dtype=torch.float64, device=self.device)
        d = torch.empty(self.O, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().nb_world_read_behaviors(self._handle, self._envs, C.c_void_p(g.data_ptr()), C.c_void_p(d.data_ptr()), self._stream()))
        return g, d

    def map_bounces(self) -> torch.Tensor:
        """(O,) int32 on the device: per obstacle, the steps in which a map that blocks obstacles turned its move back (0 for
        obstacles of scenes whose map does not block them).  Needs scenes with ``"blocks_obstacles": True``; a copy enqueued on the
        current stream."""
        if not getattr(self, "map_contact", False):
            raise ValueError("no scene's map blocks obstacles (\"blocks_obstacles\": True)")
        out = torch.empty(self.O, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().nb_world_read_map_contact(self._handle, self.O, C.c_void_p(out.data_ptr()), self._stream()))
        return out

    def obstacle_bounces(self) -> torch.Tensor:
        """(O,) int32 on the device: per obstacle, the steps in which its move would have touched another obstacle and was turned
        back (0 for obstacles of scenes without obstacle contact).  Needs scenes with ``"obstacle_contact": True``; a copy enqueued on
        the current stream."""
        if not getattr(self, "obstacle_contact", False):
            raise ValueError("no scene has obstacle contact (\"obstacle_contact\": True)")
        out = torch.empty(self.O, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().nb_world_read_obstacle_contact(self._handle, self.O, C.c_void_p(out.data_ptr()), self._stream()))
        return out

    # ---- actuation limits and noise -----------------------------------------------------------------------------------------
    def set_actuation(self, limits, seed: int = 0):
        """Actuation limits and motion noise per robot type (module docstring): ``limits`` one dict per robot type with the keys
        vel_min, vel_max, acce, alpha (defaults ACTUATION_DEFAULTS), ``seed`` the motion noise's.  Needs scenes; kept by
        set_scenes and set_episodes, which zero every robot's cmd_prev."""
        rows = pack_actuation(limits, self.robots)
        if self._rows is None:
            raise ValueError("set_actuation needs scenes (set_scenes or set_episodes first)")
        per_type = (_lib.WorldActuation * len(rows))()
        for t, r in enumerate(rows):
            per_type[t].vel_min[:] = r[0:2].tolist(); per_type[t].vel_max[:] = r[2:4].tolist()
            per_type[t].acce[:] = r[4:6].tolist(); per_type[t].alpha[:] = r[6:10].tolist()
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().nb_world_set_actuation(self._handle, len(rows), per_type, C.c_uint64(int(seed))))
        self.actuation = rows

    def set_lidar_noise(self, range_std: float, range_min: float = None, seed: int = 0):
        """Lidar range noise (module docstring): a hit reports clamp(t + range_std z, range_min, range_max); ``range_min`` defaults
        to the lidar's.  range_std 0 turns it off.  Kept by set_scenes and set_episodes."""
        range_min = self.scan_dict["range_min"] if range_min is None else float(range_min)
        check_lidar_noise(float(range_std), range_min, self.scan_dict["range_max"])
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().nb_world_set_lidar_noise(self._handle, C.c_double(range_min), C.c_double(float(range_std)),
                                                            C.c_uint64(int(seed))))

    def commands(self) -> torch.Tensor:
        """(rows, 2) float64 on the device: every robot's cmd_prev, the last command after the actuation limits (zeros without
        set_actuation).  Rows are the environments' robots (N), in episode mode the scenes' own rows (S K).  A copy enqueued on the
        current stream."""
        rows = self.N if self.S is None else self.S * self.K
        out = torch.empty((rows, 2), dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().nb_world_read_commands(self._handle, rows, C.c_void_p(out.data_ptr()), self._stream()))
        return out

    def _read(self, states=None, obstacles=None, collided=None, arrived=None, rows=None):
        p = lambda t: C.c_void_p(0 if t is None else t.data_ptr())
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().nb_world_read_state(self._handle, rows or self.N, p(states), p(obstacles), p(collided), p(arrived),
                                                       self._stream()))

    # ---- continuous episodes ------------------------------------------------------------------------------------------------
    def set_episodes(self, scenes, slots: int, max_steps: int, seed: int = 0, map_window: float = 1.0):
        """Uploads a bank of S = len(scenes) <= num_envs scenes (exactly as set_scenes would for S environments: behaviours keyed by
        ``seed``, fleets, maps with ``map_window``) and runs it through ``slots`` slots (nb_world_set_episodes): slot b starts on scene
        b, and when a slot's episode ends (every robot collided or arrived, or ``max_steps`` steps) it takes the next unstarted scene on
        the device, in ascending slot and scene order; once the bank is exhausted it goes idle.  Afterwards ``N`` is slots K: scan,
        step, ``states`` and ``flags`` are slot rows (robot k of slot b at row b K + k), ``rows_of_type`` gives slot rows too, and
        ``episodes()`` the per-scene results.  Every scene of the bank needs the same K, and robot k the same type in every scene.
        set_scenes leaves episode mode."""
        check_bank(scenes, slots, max_steps, self.config.max_envs)
        rtype = pack_robot_types(scenes)
        S, K = len(scenes), fleet_size(scenes)
        _lib.check(_lib.load().nb_world_check_episodes(C.byref(self.config), S, K, C.c_void_p(rtype.ctypes.data), int(slots), int(max_steps)))
        self._upload(scenes, seed, map_window)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().nb_world_set_episodes(self._handle, int(slots), int(max_steps)))
        self.S, self.slots, self.N, self.max_steps = S, int(slots), int(slots) * K, int(max_steps)
        slot_types = np.tile(rtype[:K], int(slots))  # robot k keeps its type in every scene
        self._rows = [torch.from_numpy(np.flatnonzero(slot_types == i)).to(self.device) for i in range(len(self.robots))]

    def _read_episodes(self, **out):
        names = ("collided", "arrived", "arrive_step", "min_clearance", "end_step", "reason", "slot", "scene_of", "reset", "finished")
        if self.S is None:
            raise ValueError("not in episode mode (set_episodes)")
        p = lambda t: C.c_void_p(0 if t is None else t.data_ptr())
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().nb_world_read_episodes(self._handle, self.S, *[p(out.get(n)) for n in names], self._stream()))

    def slot_scenes(self):
        """(scene_of, reset) (slots,) int32 on the device: the scene each slot runs and 1 where a slot has just taken a new scene (every
        slot right after set_episodes) -- PlannerBatch.forward's ``scene_of`` / ``reset``.  Copies enqueued on the current stream."""
        sc, rs = (torch.empty(self.slots, dtype=torch.int32, device=self.device) for _ in range(2))
        self._read_episodes(scene_of=sc, reset=rs)
        return sc, rs

    def finished(self) -> torch.Tensor:
        """(1,) int32 on the device: the episodes ended so far."""
        f = torch.empty(1, dtype=torch.int32, device=self.device)
        self._read_episodes(finished=f)
        return f

    def episodes(self) -> dict:
        """The per-scene results, on the device: per robot of a scene (S K rows, scene s's robot k at s K + k) collided, arrived (bool,
        the flags at the episode's end), steps_to_arrive (int32, -1 = not arrived: rollout's definition) and min_clearance (float32, the
        smallest clearance over the episode's steps); per scene (S) end_step (int32, 0 while running), reason (int32: 0 while running,
        1 every robot collided or arrived, 2 max_steps reached) and slot (int32, the slot that ran it)."""
        SK, S, dev = self.S * self.K, self.S, self.device
        out = dict(collided=torch.empty(SK, dtype=torch.int32, device=dev), arrived=torch.empty(SK, dtype=torch.int32, device=dev),
                   arrive_step=torch.empty(SK, dtype=torch.int32, device=dev), min_clearance=torch.empty(SK, dtype=torch.float32, device=dev),
                   end_step=torch.empty(S, dtype=torch.int32, device=dev), reason=torch.empty(S, dtype=torch.int32, device=dev),
                   slot=torch.empty(S, dtype=torch.int32, device=dev))
        self._read_episodes(**out)
        return dict(collided=out["collided"].bool(), arrived=out["arrived"].bool(), steps_to_arrive=out["arrive_step"], min_clearance=out["min_clearance"],
                    end_step=out["end_step"], reason=out["reason"], slot=out["slot"])

    def scene_states(self):
        """(states (S K,3) float64, collided, arrived (S K,) int32) of the bank's own rows: a scene's final state once its episode has
        ended (nb_world_read_state with N = S K)."""
        SK = self.S * self.K
        s = torch.empty((SK, 3), dtype=torch.float64, device=self.device)
        c, a = (torch.empty(SK, dtype=torch.int32, device=self.device) for _ in range(2))
        self._read(states=s, collided=c, arrived=a, rows=SK)
        return s, c, a

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
        index of the object each beam hit within its environment (obstacles, then robot j as O_b + j, then the environment's map as
        O_b + K, which reports velocity 0), -1 on a miss (N,R) int32.  Passing ``velocity`` selects
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


def check_bank(scenes, slots: int, max_steps: int, max_envs: int):
    """The refusals of WorldBatch.set_episodes on the Python side (ValueError naming the scene and robot): 1 <= S = len(scenes) <=
    max_envs, 1 <= slots <= S, max_steps >= 1, every scene with the K of scene 0 and robot k of every scene with the type of robot k
    of scene 0 (nb_world_check_episodes repeats the last on the packed types)."""
    S = len(scenes)
    if not 1 <= S <= max_envs:
        raise ValueError(f"a bank of S = {S} scenes outside [1, max_envs = {max_envs}]")
    if not 1 <= int(slots) <= S:
        raise ValueError(f"slots = {slots} outside [1, S = {S}]")
    if int(max_steps) < 1:
        raise ValueError(f"max_steps = {max_steps} must be >= 1")
    robots = [sc["robots"] if "robots" in sc else [sc] for sc in scenes]
    for s, rb in enumerate(robots):
        if len(rb) != len(robots[0]):
            raise ValueError(f"scene {s} has {len(rb)} robots but scene 0 has {len(robots[0])} (every scene of a bank needs the same K)")
        for k, r in enumerate(rb):
            t, t0 = int(r.get("type", 0)), int(robots[0][k].get("type", 0))
            if t != t0:
                raise ValueError(f"scene {s}, robot {k}: type {t} but robot {k} of scene 0 has type {t0} (a robot keeps its type in every "
                                 "scene of a bank)")


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


def run_episodes(planner, world: WorldBatch, blind: bool = False, velocities: bool = True, check_every: int = 16):
    """The loop of ``rollout`` over a bank in episode mode (WorldBatch.set_episodes): scan -> planner.forward (with the world's
    ``scene_of`` / ``reset``, so that a slot's planner state starts afresh with each scene and steps that scene's path) -> step (whose
    advance kernel ends episodes and hands out the next scenes), until every scene has finished.  ``planner`` holds the bank's paths
    (PlannerBatch.load_bank / MixedPlanner.load_bank).  ``blind`` and ``velocities`` as in rollout.  Every ``check_every`` steps
    the finished count is read to the host: the loop's only host synchronisation, so idle slots cost a planner call for at most
    ``check_every`` steps after the last episode ends.  Returns WorldBatch.episodes() plus ``steps`` (the loop's step count)."""
    if world.S is None:
        raise ValueError("run_episodes needs a world in episode mode (WorldBatch.set_episodes)")
    check_every = max(1, int(check_every))
    k = 0
    while True:
        episode_steps(planner, world, check_every, blind=blind, velocities=velocities)
        k += check_every
        if int(world.finished().item()) >= world.S:  # the host synchronisation
            break
    out = world.episodes()
    out["steps"] = k
    return out


def episode_steps(planner, world: WorldBatch, steps: int, blind: bool = False, velocities: bool = True):
    """``steps`` steps of run_episodes' loop (scan -> forward with scene_of / reset -> step), without a host synchronisation."""
    N, dev = world.N, world.device
    if blind:
        blind_ranges = torch.full((N, world.R), world.scan_dict["range_max"], dtype=torch.float32, device=dev)
        blind_vel = torch.zeros((N, 2, world.R), dtype=torch.float32, device=dev)
        blind_scan = dict(world.scan_dict)
    for _ in range(steps):
        scene_of, reset = world.slot_scenes()
        ranges, vel, scan = (blind_ranges, blind_vel, blind_scan) if blind else world.scan()
        action, _ = planner.forward(world.states, ranges, scan, scan_offset=world.scan_offset, scan_velocity=vel if velocities else None,
                                    scene_of=scene_of, reset=reset)
        world.step(action)


class MixedPlanner:
    """One PlannerBatch per kind of robot behind a single ``forward``: ``groups`` is [(planner, rows), ...], each planner driving
    the world rows ``rows`` (WorldBatch.rows_of_type; together every row exactly once).  ``forward`` gathers each kind's states,
    scans and scan velocities, calls its planner and scatters the actions into one (N, 2) tensor, each kind's in its own convention
    (omni: (vx, vy)); it enqueues on the current stream without a host synchronisation, so ``rollout(MixedPlanner(...), world, ...)``
    runs a mixed world.  Returns (action, [info of each planner])."""

    def __init__(self, groups):
        self.groups = []
        for pl, rows in groups:
            rows = torch.as_tensor(rows, dtype=torch.int64).to(pl.device)
            if len(rows) != pl.B:
                raise ValueError(f"a planner of {pl.B} robots was given {len(rows)} rows")
            self.groups.append((pl, rows))
        self.N = sum(len(r) for _, r in self.groups)
        self.device = self.groups[0][0].device
        seen = torch.cat([r.to(self.device) for _, r in self.groups]).sort().values.cpu()  # once, at construction
        if not torch.equal(seen, torch.arange(self.N)):
            raise ValueError("the groups' rows must cover 0..N-1 exactly once")

    def forward(self, states, ranges=None, scan: dict = None, scan_offset=(0.0, 0.0, 0.0), scan_velocity=None, **kw):
        states = torch.as_tensor(states).reshape(self.N, 3)
        action = torch.empty((self.N, 2), dtype=torch.float32, device=self.device)
        infos = []
        for pl, rows in self.groups:
            pick = lambda t: None if t is None else t.index_select(0, rows)
            a, info = pl.forward(pick(states), pick(ranges), scan, scan_offset=scan_offset, scan_velocity=pick(scan_velocity), **kw)
            action.index_copy_(0, rows, a)
            infos.append(info)
        return action, infos

    def load_bank(self, scenes):
        """Each kind's PlannerBatch.load_bank with its robots' paths of the bank (scene_paths(scenes, type=i), i the kind's place in
        ``groups``): kind i's slot rows b K_i + m then step path row scene_of[b] K_i + m, its m-th robot of scene scene_of[b]."""
        for i, (pl, _) in enumerate(self.groups):
            pl.load_bank(scene_paths(scenes, type=i))

    def reset(self):
        for pl, _ in self.groups:
            pl.reset()

    def close(self):
        for pl, _ in self.groups:
            pl.close()


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


def _circumradius(ob) -> float:
    if "radius" in ob:
        return float(ob["radius"])
    v = np.asarray(ob.get("vertices", ob.get("outline")), np.float64)
    return float(np.hypot(v[:, 0], v[:, 1]).max())


CONTACT_GAP = 0.05  # m kept between the circumcircles of two obstacles placed with contact=True


def _separate(obs, b: int, seed: int, draw):
    """The ``contact=True`` placement of a builder: in list order, an obstacle whose circumcircle about its centre comes within
    CONTACT_GAP of that of an earlier one takes a new centre ``draw(rng)`` until it is clear (at most 1000 draws), from environment
    b's own contact stream (apart from the builder's streams, so the other draws do not change).  Circumcircles apart mean footprints
    apart, whatever the shapes."""
    rng = np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed, spawn_key=(b, 2))))
    placed = []
    for ob in obs:
        r = _circumradius(ob)
        for _ in range(1000):
            c = ob["center"]
            if all(math.hypot(c[0] - p["center"][0], c[1] - p["center"][1]) > r + _circumradius(p) + CONTACT_GAP for p in placed):
                break
            ob = dict(ob, center=tuple(float(v) for v in draw(rng)))
        else:
            raise ValueError(f"environment {b}: no place clear of the other obstacles after 1000 draws")
        placed.append(ob)
    return placed


def dyna_obs(num_envs: int, seed: int = 0, count: int = 20, behavior: str = "constant", contact: bool = False):
    """example/dyna_obs/diff/env.yaml: ``count`` (20) circles of radius 0.4..1.0 m placed at random in the box [10, 40]^2, goal
    threshold 0.4.  ``behavior="constant"``: each moves at a constant speed of at most 0.5 m/s in a random direction and bounces
    inside that box.  ``behavior="rvo"``: the example's reactive obstacles (EXAMPLE_RVO: vxmax = vymax = 0.5, wander, goal threshold
    0.3), starting at rest at the same centres.  The robot crosses the box: it starts at (6, y0) facing the goal (44, y1), y0, y1 in
    15..35 m, on a straight path.  ``contact=True``: the circles block each other (``"obstacle_contact": True``) and start apart, an
    overlapping circle drawn again in the box (``_separate``); at 0.5 m/s and step_time 0.1 a circle moves at most 0.05 m per step,
    well below the thinnest footprint (no swept test is needed)."""
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
        if contact:
            obs = _separate(obs, b, seed, lambda g: g.uniform(10.0, 40.0, 2))
        obs = _apply_behavior(obs, behavior)
        scenes.append(dict(obstacles=obs, bounds=(10.0, 10.0, 40.0, 40.0), start=start, goal=goal, goal_threshold=0.4,
                           path=line_path(start, goal)))
        if contact:
            scenes[-1]["obstacle_contact"] = True
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


def dyna_non_obs(num_envs: int, seed: int = 0, behavior: str = "constant", contact: bool = False):
    """example/dyna_non_obs/diff/{env,planner}.yaml: 11 obstacles, each one of the example's four shapes drawn uniformly -- the
    2 x 2 m square, a circle of r = 1.5, a circle of r = 1.0, or an outline of average radius U(0.5, 1.5) and irregularity 0.9 (how
    IR-SIM assigns a 4-entry shape list to 11 obstacles is a stated choice here).  Centres uniform in [5, 45] x [15, 35].
    ``behavior="constant"``: constant velocities (vx, vy) in U(-1, 1)^2, bouncing in that box.  ``behavior="rvo"``: the example's
    reactive obstacles (EXAMPLE_RVO), circles, squares and outlines alike, starting at rest at the same centres.  The robot starts
    at (-1, 25, 0) on the planner's line path to (50, 25), its goal, with threshold 0.4.  ``contact=True``: the obstacles block each
    other (``"obstacle_contact": True``) and start apart, an overlapping one drawn again in the box (``_separate``)."""
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
        if contact:
            obs = _separate(obs, b, seed, lambda g: g.uniform((5.0, 15.0), (45.0, 35.0)))
        obs = _apply_behavior(obs, behavior)
        scenes.append(dict(obstacles=obs, bounds=(5.0, 15.0, 45.0, 35.0), start=start, goal=goal, goal_threshold=0.4,
                           path=line_path(start, goal)))
        if contact:
            scenes[-1]["obstacle_contact"] = True
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


def mixed_swap(num_envs: int, types=(0, 1, 2), robots: int = 6, radius: float = 10.0, seed: int = 0, circles: int = 0):
    """circle_swap with robot k of type ``types[k % len(types)]`` (a WorldBatch of several robot types): the same starts, goals,
    paths and obstacles as circle_swap(num_envs, robots, radius, seed, circles).  With the default types (0, 1, 2) and the shipped
    bodies (C4's 1.6 x 2.0 m diff robot, C2's 4.6 x 1.6 m car, C5's trapezoid) six robots on the default 10 m circle start 10 m
    apart, clear of the car's 3.9 m circumradius about its rear axle; nb_world_check_fleet_ex refuses starts whose bodies meet."""
    types = tuple(int(t) for t in types)
    if not types or min(types) < 0 or max(types) >= MAX_ROBOT_TYPES:
        raise ValueError(f"types must be a non-empty sequence of 0..{MAX_ROBOT_TYPES - 1} (got {types})")
    scenes = circle_swap(num_envs, robots=robots, radius=radius, seed=seed, circles=circles)
    for sc in scenes:
        sc["robots"] = [dict(rb, type=types[k % len(types)]) for k, rb in enumerate(sc["robots"])]
    return scenes


# ---- occupancy-map scenes ----------------------------------------------------------------------------------------------------

def _layouts(num_envs: int, layouts):
    L = int(num_envs) if layouts is None else int(layouts)
    if L < 1:
        raise ValueError(f"layouts must be positive (got {L})")
    return L


def _polyline_path(points, spacing: float = 0.1) -> np.ndarray:
    """(n,4) rows [x, y, theta, gear = 1] along the polyline through ``points``, each segment at ``spacing`` with its own heading."""
    segs = [line_path(a, b, spacing) for a, b in zip(points[:-1], points[1:])]
    return np.concatenate([segs[0]] + [s[1:] for s in segs[1:]])


def _fill_rect(occ, x0, x1, y0, y1, origin, res):
    """Marks the cells of occ whose centres lie in [x0, x1] x [y0, y1]."""
    H, W = occ.shape
    i0, i1 = max(0, math.ceil((x0 - origin[0]) / res - 0.5)), min(W - 1, math.floor((x1 - origin[0]) / res - 0.5))
    j0, j1 = max(0, math.ceil((y0 - origin[1]) / res - 0.5)), min(H - 1, math.floor((y1 - origin[1]) / res - 0.5))
    if i0 <= i1 and j0 <= j1:
        occ[j0:j1 + 1, i0:i1 + 1] = True


def _maze_layout(rng, nx: int, ny: int):
    """A perfect maze on nx x ny cells by randomised depth-first search from cell (0, 0): the set of open passages
    {((a, c), (a', c'))} and the solution from (0, 0) to (nx - 1, ny - 1) as a list of cells."""
    seen, stack, parent, open_ = {(0, 0)}, [(0, 0)], {(0, 0): None}, set()
    while stack:
        a, c = stack[-1]
        nbrs = [(a + da, c + dc) for da, dc in ((1, 0), (-1, 0), (0, 1), (0, -1)) if 0 <= a + da < nx and 0 <= c + dc < ny
                and (a + da, c + dc) not in seen]
        if not nbrs:
            stack.pop()
            continue
        nxt = nbrs[int(rng.integers(len(nbrs)))]
        seen.add(nxt)
        parent[nxt] = (a, c)
        open_.add(frozenset(((a, c), nxt)))
        stack.append(nxt)
    sol, cell = [], (nx - 1, ny - 1)
    while cell is not None:  # the tree path back to the root
        sol.append(cell)
        cell = parent[cell]
    return open_, sol[::-1]


def _movers(b: int, seed: int, centres, count: int, behavior: str, contact: bool = False):
    """``count`` circles of radius U(0.3, 0.6) at centres drawn from ``centres`` (distinct while there are enough), from
    environment b's own movers stream (apart from the layout streams, so the maps do not change): behavior "constant" moves each at
    a speed U(0, 0.5) m/s in a random direction, "rvo" starts it at rest with EXAMPLE_RVO.  ``contact``: a circle that would overlap
    an earlier one takes another of ``centres`` (``_separate``)."""
    rng = np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed, spawn_key=(b, 1))))
    if not len(centres):
        raise ValueError("no free place for a moving obstacle")
    pick = rng.choice(len(centres), count, replace=count > len(centres))
    r = rng.uniform(0.3, 0.6, count)
    speed, heading = rng.uniform(0.0, 0.5, count), rng.uniform(-math.pi, math.pi, count)
    obs = [dict(center=tuple(float(v) for v in centres[pick[i]]), radius=float(r[i]),
                velocity=(speed[i] * math.cos(heading[i]), speed[i] * math.sin(heading[i]))) for i in range(count)]
    if contact:
        obs = _separate(obs, b, seed, lambda g: centres[int(g.integers(len(centres)))])
    return _apply_behavior(obs, behavior)


def maze(num_envs: int, cells=(6, 6), cell_size: float = 5.0, wall: float = 0.3, resolution: float = 0.1, seed: int = 0, layouts=None,
         movers: int = 0, behavior: str = "constant", contact: bool = False):
    """Perfect mazes on an occupancy map: ``cells`` (nx, ny) maze cells of ``cell_size`` m, carved by a randomised depth-first search
    (every cell reachable by exactly one route), rasterised at ``resolution`` with walls ``wall`` m thick centred on the closed cell
    boundaries, the outer border included.  Maze cell (a, c) is [a s, (a + 1) s] x [c s, (c + 1) s]; the map covers that area plus
    ``wall`` on every side.  The robot starts at the centre of cell (0, 0) facing along the solution; its goal is the centre of cell
    (nx - 1, ny - 1) with threshold 0.3; ``path`` is the solution through the cell centres at 0.1 m spacing (each segment's heading,
    gear 1).  ``layouts`` distinct mazes (default: one per environment), environment b taking layout b mod layouts, each seeded by
    its own child stream (``_rng(seed, layout)``); environments of one layout share its occupancy array (one copy on the device).
    ``movers`` > 0: that many circles of radius U(0.3, 0.6) m at the centres of maze cells other than the start cell and its eight
    neighbours, moving at U(0, 0.5) m/s in a random direction (``behavior="constant"``) or starting at rest as the examples' reactive
    obstacles (``"rvo"``, EXAMPLE_RVO: wander in the maze's rectangle), drawn per environment; the map then blocks obstacles
    (``"blocks_obstacles": True``).  The speeds need step_time * 0.5 m/s (constant) or * 0.71 m/s (rvo) below ``resolution``.
    ``contact=True`` (with movers): the movers also block each other (``"obstacle_contact": True``) and start apart."""
    nx, ny = (int(v) for v in cells)
    if nx < 1 or ny < 1 or not (0.0 < wall < cell_size):
        raise ValueError("maze needs cells >= 1 and 0 < wall < cell_size")
    L = _layouts(num_envs, layouts)
    origin = (-wall, -wall)
    W, H = int(round((nx * cell_size + 2 * wall) / resolution)), int(round((ny * cell_size + 2 * wall) / resolution))
    built = []
    for lay in range(min(L, num_envs)):
        open_, sol = _maze_layout(_rng(seed, lay), nx, ny)
        occ = np.zeros((H, W), bool)
        h = wall / 2.0
        for a in range(nx + 1):  # vertical walls x = a s between (a - 1, c) and (a, c)
            for c in range(ny):
                if 0 < a < nx and frozenset(((a - 1, c), (a, c))) in open_:
                    continue
                _fill_rect(occ, a * cell_size - h, a * cell_size + h, c * cell_size - h, (c + 1) * cell_size + h, origin, resolution)
        for c in range(ny + 1):  # horizontal walls y = c s between (a, c - 1) and (a, c)
            for a in range(nx):
                if 0 < c < ny and frozenset(((a, c - 1), (a, c))) in open_:
                    continue
                _fill_rect(occ, a * cell_size - h, (a + 1) * cell_size + h, c * cell_size - h, c * cell_size + h, origin, resolution)
        pts = [((a + 0.5) * cell_size, (c + 0.5) * cell_size) for a, c in sol]
        built.append((occ, pts))
    scenes = []
    for b in range(num_envs):
        occ, pts = built[b % L]
        th = math.atan2(pts[1][1] - pts[0][1], pts[1][0] - pts[0][0]) if len(pts) > 1 else 0.0
        path = _polyline_path(pts) if len(pts) > 1 else np.array([[pts[0][0], pts[0][1], th, 1.0]])
        scenes.append(dict(obstacles=[], bounds=(0.0, 0.0, nx * cell_size, ny * cell_size), start=(pts[0][0], pts[0][1], th), goal=pts[-1],
                           goal_threshold=0.3, path=path, map=dict(occupancy=occ, origin=origin, resolution=resolution)))
        if movers > 0:
            free = [((a + 0.5) * cell_size, (c + 0.5) * cell_size) for c in range(ny) for a in range(nx) if max(a, c) > 1]
            scenes[-1]["obstacles"] = _movers(b, seed, free, int(movers), behavior, contact)
            scenes[-1]["map"]["blocks_obstacles"] = True
            if contact:
                scenes[-1]["obstacle_contact"] = True
    return scenes


def _components(free):
    """Labels of the 4-connected components of the True cells of ``free`` (-1 elsewhere) and their sizes."""
    H, W = free.shape
    lab = np.full((H, W), -1, np.int64)
    sizes = []
    for j0, i0 in zip(*np.nonzero(free)):
        if lab[j0, i0] >= 0:
            continue
        lab[j0, i0] = len(sizes)
        queue, n = [(j0, i0)], 0
        while queue:
            j, i = queue.pop()
            n += 1
            for jj, ii in ((j + 1, i), (j - 1, i), (j, i + 1), (j, i - 1)):
                if 0 <= jj < H and 0 <= ii < W and free[jj, ii] and lab[jj, ii] < 0:
                    lab[jj, ii] = len(sizes)
                    queue.append((jj, ii))
        sizes.append(n)
    return lab, sizes


def _bfs(free, start):
    """Breadth-first search over the 4-connected True cells of ``free`` from ``start`` (j, i): (distance (-1 unreached), parent)."""
    H, W = free.shape
    dist = np.full((H, W), -1, np.int64)
    parent = {start: None}
    dist[start] = 0
    queue, q = [start], 0
    while q < len(queue):
        j, i = queue[q]
        q += 1
        for jj, ii in ((j + 1, i), (j - 1, i), (j, i + 1), (j, i - 1)):
            if 0 <= jj < H and 0 <= ii < W and free[jj, ii] and dist[jj, ii] < 0:
                dist[jj, ii] = dist[j, i] + 1
                parent[(jj, ii)] = (j, i)
                queue.append((jj, ii))
    return dist, parent


def cave(num_envs: int, size=(40.0, 40.0), resolution: float = 0.1, fill: float = 0.45, seed: int = 0, layouts=None,
         coarse: float = 1.0, clearance: float = 2.0, movers: int = 0, behavior: str = "constant", contact: bool = False):
    """Caves on an occupancy map: a cellular automaton on a coarse grid of ``coarse`` m cells over ``size`` (m) -- each cell a wall
    with probability ``fill``, the border always a wall, then 5 rounds of the 4-5 rule (a cell becomes a wall when at least 5 of
    its 8 neighbours are walls, free when at most 3 are, cells past the border counting as walls) -- of which only the largest
    4-connected free region is kept free; upsampled to ``resolution``, origin (0, 0).  Start and goal are the centres of coarse
    cells whose distance to every wall cell's centre exceeds ``clearance`` + ``coarse`` (``clearance``: the robot's circumradius
    plus a margin; the default 2.0 m covers C4's 1.28 m body): the start a random such cell of the largest 4-connected group of
    them, the goal the cell of that group farthest from it by breadth-first search; ``path`` is that breadth-first path through the
    cell centres at 0.1 m spacing, the start facing along it, goal threshold 0.3.  ``layouts`` as in ``maze``.  ``movers`` and
    ``behavior`` as in ``maze``, the circles at the centres of free coarse cells whose eight neighbours are free too and that lie at
    least 4 m from the start (wander in the cave's rectangle).  ``contact`` as in ``maze``."""
    sx, sy = float(size[0]), float(size[1])
    nx, ny = int(round(sx / coarse)), int(round(sy / coarse))
    up = int(round(coarse / resolution))
    if nx < 3 or ny < 3 or up < 1 or abs(up * resolution - coarse) > 1e-9 * coarse:
        raise ValueError("cave needs at least 3 x 3 coarse cells and a coarse side that is a multiple of the resolution")
    L = _layouts(num_envs, layouts)
    built = []
    for lay in range(min(L, num_envs)):
        rng = _rng(seed, lay)
        for _ in range(64):  # a draw without a cell far enough from the walls is drawn again
            wall = rng.uniform(size=(ny, nx)) < fill
            wall[0], wall[-1], wall[:, 0], wall[:, -1] = True, True, True, True
            for _ in range(5):
                pad = np.pad(wall, 1, constant_values=True).astype(np.int64)
                n = sum(np.roll(np.roll(pad, dj, 0), di, 1) for dj in (-1, 0, 1) for di in (-1, 0, 1) if dj or di)[1:-1, 1:-1]
                wall = np.where(n >= 5, True, np.where(n <= 3, False, wall))
                wall[0], wall[-1], wall[:, 0], wall[:, -1] = True, True, True, True
            lab, sizes = _components(~wall)
            if not sizes:
                continue
            wall = lab != int(np.argmax(sizes))
            jw, iw = np.nonzero(wall)
            jf, if_ = np.nonzero(~wall)
            d = np.sqrt((jf[:, None] - jw[None]) ** 2 + (if_[:, None] - iw[None]) ** 2).min(1) * coarse
            safe = np.zeros_like(wall)
            safe[jf[d > clearance + coarse], if_[d > clearance + coarse]] = True
            slab, ssizes = _components(safe)
            if not ssizes or max(ssizes) < 2:
                continue
            group = slab == int(np.argmax(ssizes))
            cand = np.argwhere(group)
            start = tuple(int(v) for v in cand[int(rng.integers(len(cand)))])
            dist, parent = _bfs(group, start)
            goal = tuple(int(v) for v in np.unravel_index(int(np.argmax(dist)), dist.shape))
            route, cell = [], goal
            while cell is not None:
                route.append(cell)
                cell = parent[cell]
            pts = [((i + 0.5) * coarse, (j + 0.5) * coarse) for j, i in route[::-1]]
            break
        else:
            raise ValueError("cave: no layout with a start far enough from the walls (lower fill or clearance)")
        occ = np.kron(wall, np.ones((up, up), bool))
        open9 = ~np.pad(wall, 1, constant_values=True)
        open9 = np.logical_and.reduce([open9[1 + dj:1 + dj + ny, 1 + di:1 + di + nx] for dj in (-1, 0, 1) for di in (-1, 0, 1)])
        free = [((i + 0.5) * coarse, (j + 0.5) * coarse) for j, i in zip(*np.nonzero(open9))
                if math.hypot((i + 0.5) * coarse - pts[0][0], (j + 0.5) * coarse - pts[0][1]) >= 4.0]
        built.append((occ, pts, free))
    scenes = []
    for b in range(num_envs):
        occ, pts, free = built[b % L]
        th = math.atan2(pts[1][1] - pts[0][1], pts[1][0] - pts[0][0])
        scenes.append(dict(obstacles=[], bounds=(0.0, 0.0, sx, sy), start=(pts[0][0], pts[0][1], th), goal=pts[-1], goal_threshold=0.3,
                           path=_polyline_path(pts), map=dict(occupancy=occ, origin=(0.0, 0.0), resolution=resolution)))
        if movers > 0:
            scenes[-1]["obstacles"] = _movers(b, seed, free, int(movers), behavior, contact)
            scenes[-1]["map"]["blocks_obstacles"] = True
            if contact:
                scenes[-1]["obstacle_contact"] = True
    return scenes
