"""B robots, one control step, on the device: ``neupan.forward`` (neupan/neupan.py:104-167) for a batch.

    state, scan  ->  check_arrive + generate_nom_ref_state   (InitialPathBatch,   initial_path.py:68-126, 251-292)
                 ->  scan_to_point(_velocity) + decimation   (scan_to_points,     neupan.py:173-281, pan.py:171-174)
                 ->  PAN.forward                              (neupan_b200.PAN,    pan.py:109-147)
                 ->  action = first optimal velocity, zero for robots that arrived or must stop (neupan.py:114-116, 150-164)

Everything between the input tensors and the returned action stays in GPU memory.  This is an extension of the reference
API (the reference plans for one robot); the single-robot facade with the reference's exact signature is ``neupan_b200.neupan``.
Difference to B independent reference planners: PAN also runs for robots that have already arrived (their action is zeroed and
their velocity memory is kept, but PAN's stop-criterion memory of those environments advances).
"""
from __future__ import annotations

import numpy as np
import torch

from .blocks.pan import PAN
from .ipath import InitialPathBatch
from .robot import robot as Robot
from .scan import scan_to_points


class PlannerBatch:
    def __init__(self, num_envs: int, receding: int = 10, step_time: float = 0.1, ref_speed: float = 4.0, robot_kwargs: dict = None,
                 ipath_kwargs: dict = None, pan_kwargs: dict = None, adjust_kwargs: dict = None, collision_threshold: float = 0.1, device=None):
        self.B, self.T, self.dt, self.ref_speed = int(num_envs), receding, step_time, ref_speed
        self.collision_threshold = collision_threshold
        self.robot = Robot(receding, step_time, **(robot_kwargs or {}))
        pk = dict(pan_kwargs or {})
        pk["adjust_kwargs"] = adjust_kwargs
        pk.setdefault("max_envs", self.B)
        if device is not None:
            pk.setdefault("device", torch.device(device))
        self.pan = PAN(receding, step_time, self.robot, **pk)
        self.device = self.pan.device
        self._ipath_kwargs = dict(ipath_kwargs or {})
        self.ipath = self._make_ipath(self.B)
        self.cur_vel = torch.zeros(self.B, 2, receding, dtype=torch.float32, device=self.device)  # neupan.py:73
        self.info = {}

    def _make_ipath(self, max_envs: int) -> InitialPathBatch:
        ik = self._ipath_kwargs
        return InitialPathBatch(self.T, self.dt, self.robot.kinematics, self.robot.L, loop=ik.get("loop", False),
                                arrive_threshold=ik.get("arrive_threshold", 0.1), close_threshold=ik.get("close_threshold", 0.1),
                                ind_range=ik.get("ind_range", 10), arrive_index_threshold=ik.get("arrive_index_threshold", 1),
                                max_envs=max_envs, device=self.device)

    def load_bank(self, paths):
        """The initial paths of a bank of scenes for continuous episodes (WorldBatch.set_episodes, run_episodes): one per robot of
        the bank in row order (scene_paths; S K' paths when this planner drives K' robots of each of the slots), any count.  forward
        with ``scene_of`` then steps row b K' + m on path scene_of[b] K' + m."""
        if len(paths) > self.ipath.max_envs:
            self.ipath.close()
            self.ipath = self._make_ipath(len(paths))
        self.ipath.set_initial_paths(paths)

    def set_initial_paths(self, paths):
        """neupan.set_initial_path (neupan.py:296-303) for every robot."""
        if len(paths) != self.B:
            raise ValueError(f"expected {self.B} paths, got {len(paths)}")
        self.ipath.set_initial_paths(paths)

    def reset(self):
        """neupan.reset (neupan.py:287-294)."""
        self.ipath.reset()
        self.cur_vel.zero_()

    def forward(self, states, ranges=None, scan: dict = None, scan_offset=(0.0, 0.0, 0.0), angle_range=(-np.pi, np.pi), down_sample: int = 1,
                scan_velocity=None, points=None, point_velocities=None, num_points=None, scene_of=None, reset=None):
        """states (B,3).  Obstacles either as lidar scans (``ranges`` (B,R) + the ``scan`` dict, optional ``scan_velocity``
        (B,2,R)) or as ready point clouds (``points`` (B,2,N), ``point_velocities``, ``num_points``).
        Continuous episodes (after load_bank): ``scene_of`` (slots,) int32 on the device, the scene each slot runs, with B = slots K';
        row b K' + m steps path scene_of[b] K' + m.  ``reset`` (slots,) int32: where it is 1 the slot's K' rows start afresh -- cur_vel
        zeroed and PAN's stop-criterion memory forgotten (nb_pan_reset_envs_async) -- with device ops only.
        Returns (action (B,2) float32 on the device, info)."""
        states = torch.as_tensor(states).reshape(self.B, 3).to(self.device, torch.float64)
        env_index = None
        if scene_of is not None:
            scene_of = torch.as_tensor(scene_of, device=self.device)
            if self.B % scene_of.numel():
                raise ValueError(f"{self.B} planners do not split into {scene_of.numel()} slots")
            k = self.B // scene_of.numel()
            env_index = (scene_of.to(torch.int32)[:, None] * k + torch.arange(k, dtype=torch.int32, device=self.device)).reshape(-1)
        if reset is not None:
            rows = torch.as_tensor(reset, device=self.device).to(torch.int32).repeat_interleave(self.B // reset.numel())
            self.cur_vel = torch.where(rows[:, None, None] != 0, 0.0, self.cur_vel)
            self.pan.reset_envs(rows)
        nom_s, nom_u, ref_s, ref_us, arrived = self.ipath.step(states, self.cur_vel, self.ref_speed, env_index=env_index)
        if ranges is not None:
            points, point_velocities, num_points = scan_to_points(states, ranges, scan, scan_offset, angle_range, down_sample,
                                                                  max_points=self.pan.dune_max_num, velocity=scan_velocity, device=self.device)
        with torch.no_grad():  # batched control is inference; tune parameters through neupan / PAN (differentiable mode) instead
            opt_s, opt_u, opt_d = self.pan(nom_s, nom_u, ref_s, ref_us, points, point_velocities, num_points)
        arrive = arrived.bool()
        md = self.pan.min_distance
        md = md if torch.is_tensor(md) else torch.full((self.B,), float(md), device=self.device)
        stop = (md < self.collision_threshold) & ~arrive                      # neupan.check_stop (neupan.py:169-170)
        self.cur_vel = torch.where(arrive[:, None, None], self.cur_vel, opt_u)  # an arrived robot returns before PAN (neupan.py:114-116)
        action = opt_u[:, :, 0].clone()
        if self.robot.kinematics == "omni":  # neupan.py:155-163
            v, th = action[:, 0].clone(), action[:, 1].clone()
            action = torch.stack([v * torch.cos(th), v * torch.sin(th)], 1)
        action[arrive | stop] = 0.0
        self.info = dict(arrive=arrive, stop=stop, state_tensor=opt_s, vel_tensor=opt_u, distance_tensor=opt_d, ref_state_tensor=ref_s,
                         ref_speed_tensor=ref_us, nom_state_tensor=nom_s, min_distance=md, num_points=num_points)
        return action, self.info

    def close(self):
        self.ipath.close()
        self.pan.close()
