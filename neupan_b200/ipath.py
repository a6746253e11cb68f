"""Batched initial-path stepping on the GPU (SURVEY 8f "next" row 1).

``InitialPathBatch`` holds the naive initial paths of B environments and performs, per control step and for all of them
at once, what ``neupan.forward`` asks of ``InitialPath`` before PAN (neupan/neupan.py:114-121):
``check_arrive`` (neupan/blocks/initial_path.py:251-292) and ``generate_nom_ref_state`` (:68-126).  Its outputs are
``PAN.forward``'s ``nom_s, nom_u, ref_s, ref_us`` on the device.  Paths enter as explicit point lists like through
``neupan.set_initial_path`` (neupan.py:296-303); generating curves from waypoints stays with the host-side
``neupan_b200.blocks.InitialPath``.  There is no CPU implementation of the stepping here.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from . import _lib


def _as_rows(path) -> np.ndarray:
    """list of (4,1) arrays / (n,4) array -> (n,4) float64 rows [x, y, theta, gear]"""
    if isinstance(path, np.ndarray) and path.ndim == 2 and path.shape[1] == 4:
        return np.ascontiguousarray(path, dtype=np.float64)
    return np.ascontiguousarray(np.hstack([np.asarray(p, dtype=np.float64).reshape(4, 1) for p in path]).T)


class InitialPathBatch:
    def __init__(self, receding: int, step_time: float, kinematics: str, wheelbase: float | None = None, loop: bool = False,
                 arrive_threshold: float = 0.1, close_threshold: float = 0.1, ind_range: int = 10, arrive_index_threshold: int = 1,
                 max_envs: int = 1, device=None):
        if kinematics not in _lib.NB_KIN:
            raise ValueError("kinematics currently only supports diff, acker or omni")
        if not torch.cuda.is_available():
            raise RuntimeError("neupan_b200.InitialPathBatch needs a CUDA device (no CPU fallback)")
        self.T, self.dt = int(receding), float(step_time)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        cfg = _lib.IpathConfig(receding=self.T, kinematics=_lib.NB_KIN[kinematics], loop=int(bool(loop)), ind_range=int(ind_range),
                               arrive_index_threshold=int(arrive_index_threshold), max_envs=int(max_envs), device=self.device.index or 0,
                               step_time=self.dt, wheelbase=float(wheelbase or 0.0), arrive_threshold=float(arrive_threshold),
                               close_threshold=float(close_threshold))
        self._handle = C.c_void_p()
        _lib.check(_lib.load().nb_ipath_create(C.byref(cfg), C.byref(self._handle)))
        self.B, self.P, self.max_envs = 0, 0, int(max_envs)

    def close(self):
        if getattr(self, "_handle", None):
            _lib.load().nb_ipath_destroy(self._handle)
            self._handle = None

    __del__ = close

    # ---- InitialPath.set_initial_path for every environment (initial_path.py:128-164, 294-317) --------------------
    def set_initial_paths(self, paths):
        rows = [_as_rows(p) for p in paths]
        pts, curve_begin, env_curve_begin, interval = [], [0], [0], []
        for r in rows:
            n = r.shape[0]
            if n < 1:
                raise ValueError("a path needs at least one point")
            dist = 0.0
            for i in range(n - 1):  # cal_average_interval (:146-164)
                dist += math.hypot(r[i + 1, 0] - r[i, 0], r[i + 1, 1] - r[i, 1])
            interval.append(dist / (n - 1) if n >= 2 else 0.0)
            cuts = [0] + [i for i in range(1, n) if r[i, 3] != r[i - 1, 3]] + [n]  # split_path_with_gear (:294-317)
            for a, b in zip(cuts, cuts[1:]):
                curve_begin.append(curve_begin[-1] + (b - a))
            env_curve_begin.append(len(curve_begin) - 1)
            pts.append(r)
        pts = np.ascontiguousarray(np.vstack(pts))
        cb, eb, iv = np.asarray(curve_begin, np.int32), np.asarray(env_curve_begin, np.int32), np.asarray(interval, np.float64)
        self.B, self.P = len(rows), pts.shape[0]
        hp = lambda a: C.c_void_p(a.ctypes.data)
        _lib.check(_lib.load().nb_ipath_set_paths(self._handle, self.B, hp(pts), self.P, hp(cb), len(cb) - 1, hp(eb), hp(iv)))
        self.interval = iv

    # ---- one control step (neupan.py:114-121) ---------------------------------------------------------------------
    def step(self, states, cur_vel, ref_speed: float, env_index=None):
        """states (B,3) [x, y, theta]; cur_vel (B,2,T).  Returns (nom_s (B,3,T+1), nom_u (B,2,T), ref_s (B,3,T+1),
        ref_us (B,T), arrived (B,) int32) on the GPU: the arguments of PAN.forward plus the arrive flags.  ``env_index`` (B,) int32
        on the device (nb_ipath_step_ex): row b steps path and state env_index[b] of the paths set, B = len(env_index)."""
        dev, T = self.device, self.T
        B = self.B if env_index is None else int(env_index.numel())
        if env_index is not None:
            env_index = env_index.to(device=dev, dtype=torch.int32).contiguous()
        states = torch.as_tensor(states).reshape(B, 3).to(device=dev, dtype=torch.float64).contiguous()
        cur_vel = torch.as_tensor(cur_vel).reshape(B, 2, T).to(device=dev, dtype=torch.float32).contiguous()
        mk = lambda *s, dtype=torch.float32: torch.empty(s, dtype=dtype, device=dev)
        nom_s, nom_u, ref_s, ref_us, arrived = mk(B, 3, T + 1), mk(B, 2, T), mk(B, 3, T + 1), mk(B, T), mk(B, dtype=torch.int32)
        ptr = lambda t: C.c_void_p(t.data_ptr())
        with torch.cuda.device(dev):
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            if env_index is None:
                _lib.check(_lib.load().nb_ipath_step(self._handle, B, ptr(states), ptr(cur_vel), float(ref_speed), ptr(nom_s), ptr(nom_u),
                                                     ptr(ref_s), ptr(ref_us), ptr(arrived), stream))
            else:
                _lib.check(_lib.load().nb_ipath_step_ex(self._handle, B, ptr(env_index), ptr(states), ptr(cur_vel), float(ref_speed), ptr(nom_s),
                                                        ptr(nom_u), ptr(ref_s), ptr(ref_us), ptr(arrived), stream))
        return nom_s, nom_u, ref_s, ref_us, arrived

    def reset(self):
        """neupan.reset (neupan.py:287-294)."""
        with torch.cuda.device(self.device):
            stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            _lib.check(_lib.load().nb_ipath_reset_async(self._handle, stream))

    def read_state(self):
        dev, B = self.device, self.B
        ci, pi, af = (torch.empty(B, dtype=torch.int32, device=dev) for _ in range(3))
        pts = np.empty((self.P, 4), np.float64)
        with torch.cuda.device(dev):
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(_lib.load().nb_ipath_read_state(self._handle, B, C.c_void_p(ci.data_ptr()), C.c_void_p(pi.data_ptr()), C.c_void_p(af.data_ptr()),
                                                       C.c_void_p(pts.ctypes.data), stream))
        return dict(curve_index=ci, point_index=pi, arrive_flag=af, points=pts)
