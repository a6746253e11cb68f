"""PAN: the drop-in boundary of the hot path (mirrors neupan/blocks/pan.py:27-274).

Same constructor and ``forward(nom_s, nom_u, ref_s, ref_us, obs_points=None, point_velocities=None)
-> (nom_s, nom_u, nom_distance)`` as the reference; every tensor may carry a leading batch axis B
of independent environments (the reference is the unbatched case).  All computation is done by
libneupan_b200.so (sm_90a CUDA) through its C ABI -- there is no torch / CPU compute path:

* CUDA tensors in  -> ``nb_pan_forward`` on torch's current stream, CUDA tensors out (no sync);
* CPU tensors in   -> ``nb_pan_forward_host`` (H2D, compute, D2H in one call), CPU tensors out,
                      which is what neupan.forward does around PAN (neupan/neupan.py:123-135).

Extra keyword arguments (extensions): ``device`` (CUDA device that computes, default current),
``max_envs`` / ``max_points`` (initial capacities; the native handle is re-created when a call
exceeds them).
"""
from __future__ import annotations

import ctypes as C
from math import inf
from typing import Optional

import numpy as np
import torch

from .. import _lib
from ..configuration import tensor_to_np
from ..util import decimation_indices
from .dune import DUNE
from .nrmp import NRMP


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


class _PanSolve(torch.autograd.Function):
    """Differentiable PAN.forward: the forward is the native nb_pan_forward in differentiable mode, the backward is
    nb_pan_backward (adjoint solves of the K NRMP programs on the device) -- what CvxpyLayer's backward does in the reference
    (nrmp.py:144), reaching the leaves q_s, p_u, eta, d_max, d_min of NRMP.adjust_parameters (nrmp.py:79-104)."""

    @staticmethod
    def forward(ctx, pan, run, ref_s, ref_us, q_s, p_u, *dist_params):
        out_s, out_u, out_d = run()
        ctx.pan, ctx.ref_s, ctx.ref_us = pan, ref_s, ref_us
        ctx.q_shape, ctx.n_dist = tuple(q_s.shape), len(dist_params)
        ctx.out_device = out_s.device
        ctx.forward_id = pan._forward_id
        return out_s, out_u, out_d

    @staticmethod
    def backward(ctx, g_s, g_u, g_d):
        pan = ctx.pan
        if pan._forward_id != ctx.forward_id:
            raise RuntimeError("neupan_b200.PAN: backward() of an earlier forward -- the native adjoint records belong to the latest forward only "
                               "(call loss.backward() before the next planner step, as example/LON does)")
        dev = pan.device
        B = ctx.ref_s.shape[0]
        prep = lambda t: None if t is None else t.detach().to(device=dev, dtype=torch.float32).contiguous()
        g_s, g_u = prep(g_s), prep(g_u)
        g_d = None if g_d is None else prep(g_d).reshape(B, -1)
        ref_s, ref_us = prep(ctx.ref_s), prep(ctx.ref_us)
        gth = torch.empty((B, 7), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(_lib.load().nb_pan_backward(pan._handle, B, _ptr(ref_s), _ptr(ref_us), _ptr(g_s), _ptr(g_u), _ptr(g_d), _ptr(gth), stream))
        pan.last_grad_theta = gth  # (B, 7) per-environment gradients [q0, q1, q2, p_u, eta, d_max, d_min] (diagnostics / tests)
        g = gth.sum(0).to("cpu")  # the adjust parameters are shared by the batch
        gq = g[0:3].reshape(3, 1) if ctx.q_shape == (3, 1) else g[0:3].sum().reshape(ctx.q_shape)
        grads = [gq, g[3].reshape(()), g[4].reshape(()), g[5].reshape(()), g[6].reshape(())]
        return (None, None, None, None, *grads[:2 + ctx.n_dist])


class PAN(torch.nn.Module):
    def __init__(self, receding=10, step_time=0.1, robot=None, iter_num=2, dune_max_num=100, nrmp_max_num=10, dune_checkpoint=None,
                 iter_threshold=0.1, adjust_kwargs=None, train_kwargs=None, **kwargs) -> None:
        super().__init__()
        adjust_kwargs = dict() if adjust_kwargs is None else adjust_kwargs
        train_kwargs = dict() if train_kwargs is None else train_kwargs
        self.robot = robot
        self.T = receding
        self.dt = step_time
        self.iter_num = iter_num
        self.iter_threshold = iter_threshold
        self.nrmp_layer = NRMP(
            receding, step_time, robot, nrmp_max_num,
            eta=adjust_kwargs.get("eta", 10.0), d_max=adjust_kwargs.get("d_max", 1.0), d_min=adjust_kwargs.get("d_min", 0.1),
            q_s=adjust_kwargs.get("q_s", 1.0), p_u=adjust_kwargs.get("p_u", 1.0), ro_obs=adjust_kwargs.get("ro_obs", 400),
            bk=adjust_kwargs.get("bk", 0.1), solver=adjust_kwargs.get("solver", "ECOS"))
        self.no_obs = nrmp_max_num == 0 or dune_max_num == 0  # pan.py:85
        self.nrmp_max_num = nrmp_max_num
        self.dune_max_num = dune_max_num
        self.dune_layer = None if self.no_obs else DUNE(receding, dune_checkpoint, robot, dune_max_num, train_kwargs)
        self.printed = False

        dev = kwargs.get("device", None)
        if dev is None:
            dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cuda", 0)
        dev = torch.device(dev)
        if dev.type != "cuda":
            dev = torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)
        self.device = torch.device("cuda", dev.index if dev.index is not None else 0)
        self._handle = None
        # env sub-batches pipelined on internal streams (1 = off; batches below 64 per part are never split): the stragglers of one half's NRMP
        # launch and the small kernels between the big ones run under the other half's DUNE pass
        self.overlap = int(kwargs.get("overlap", 2))
        self.nrmp_warm = int(kwargs.get("nrmp_warm", 0))  # 1 = NRMP solves of PAN iterations k > 0 start from iteration k-1's solution (fewer IPM iterations on average, but stragglers: DESIGN.md 3.2)
        # 4 = screening pipeline (default: interval pass + exact wgmma network on the candidates, bit-identical to 2), 2 = the exact wgmma
        # network on every point; the handle refuses any other value
        self.dune_kernel = int(kwargs.get("dune_kernel", 4))
        # with dune_kernel = 4: the screening pass on mma.sync (1, default; clouds of <= 1024 points) or wgmma (0); PAN iterations k > 0
        # keep the step-0 items of iteration 0 (1, default: nom_s[:, 0] is the fixed initial state) or re-evaluate them (0).  Same results.
        self.dune_screen_mma = int(kwargs.get("dune_screen_mma", 1))
        self.dune_skip_t0 = int(kwargs.get("dune_skip_t0", 1))
        # with the mma.sync screen: look the screened distances up in the handle's distance table (1) or run the screening network on every
        # point (0).  Same results.  None keeps the handle's default (1, or NB_SCREEN_TABLE=0/1).
        self.dune_screen_table = kwargs.get("dune_screen_table")
        self._cap = (max(1, int(kwargs.get("max_envs", 1))), max(1, int(kwargs.get("max_points", max(1, dune_max_num)))))
        self._forward_id = 0
        self._differentiable = None  # last NB_OPT_DIFFERENTIABLE value pushed to the handle
        self._sent = None  # (adjust version, iter_num, iter_threshold) last pushed to the handle
        self._last = None  # bookkeeping of the last forward (for the lazy properties)

    # ------------------------------------------------------------------ native handle
    def _config(self, max_envs: int, max_points: int) -> _lib.PanConfig:
        rb, nl = self.robot, self.nrmp_layer
        cfg = _lib.PanConfig()
        cfg.receding, cfg.kinematics = int(self.T), _lib.NB_KIN[rb.kinematics]
        cfg.edge_dim = int(np.asarray(rb.G).shape[0])
        cfg.iter_num, cfg.nrmp_max_num = int(self.iter_num), (0 if self.no_obs else int(self.nrmp_max_num))
        cfg.max_envs, cfg.max_points, cfg.device = int(max_envs), int(max_points), int(self.device.index)
        cfg.iter_threshold = float(self.iter_threshold)
        cfg.step_time = float(self.dt)
        cfg.wheelbase = float(rb.L) if rb.L is not None else 0.0
        ms, ma = np.asarray(rb.max_speed, float).reshape(-1), np.asarray(rb.max_acce, float).reshape(-1)
        cfg.max_speed[0], cfg.max_speed[1] = float(ms[0]), float(ms[1])
        cfg.max_acce[0], cfg.max_acce[1] = float(ma[0]), float(ma[1])
        cfg.ro_obs, cfg.bk = float(nl.ro_obs), float(nl.bk)
        q = nl.q_vector()
        cfg.q_s[0], cfg.q_s[1], cfg.q_s[2] = float(q[0]), float(q[1]), float(q[2])
        cfg.p_u, cfg.eta = float(nl.p_u.detach()), float(nl.eta.detach())
        cfg.d_max, cfg.d_min = float(nl.d_max.detach()), float(nl.d_min.detach())
        return cfg

    def _ensure_handle(self, B: int, N: int):
        lib = _lib.load()
        cap_b, cap_n = self._cap
        wv = getattr(self.dune_layer, "weights_version", 0) if self.dune_layer is not None else 0
        if self._handle is not None and wv != getattr(self, "_weights_version", 0):
            self.close()  # DUNE.train_dune produced new weights: rebuild the native weight images
        self._weights_version = wv
        if self._handle is not None and B <= cap_b and N <= cap_n:
            return lib
        if self._handle is not None:
            # the stop criterion's memory (PAN.current_nom_values, pan.py:100-105) lives in the native handle and is dropped here
            print(f"neupan_b200.PAN: capacity grows to max_envs={max(cap_b, B)}, max_points={max(cap_n, N)}; the native handle is re-created "
                  "and the stop-criterion state of all environments is reset (pass max_envs / max_points up front to avoid this)")
        self.close()
        cap_b, cap_n = max(cap_b, B), max(cap_n, N)
        cfg = self._config(cap_b, cap_n)
        handle = C.c_void_p()
        if self.no_obs:
            w = G = h = None
            nw = 0
        else:
            w = _lib.pack_weights(self.dune_layer.model.state_dict())
            G = np.ascontiguousarray(np.asarray(self.robot.G), dtype=np.float32)
            h = np.ascontiguousarray(np.asarray(self.robot.h), dtype=np.float32).reshape(-1)
            nw = w.size
        _lib.check(lib.nb_pan_create(C.byref(cfg), None if w is None else w.ctypes.data, nw,
                                     None if G is None else G.ctypes.data, None if h is None else h.ctypes.data, C.byref(handle)))
        self._handle, self._cap = handle, (cap_b, cap_n)
        if not self.no_obs:
            if self.dune_screen_table is not None:  # before the kernel: selecting the screening pipeline builds the table when it is on
                _lib.check(lib.nb_pan_set_option(handle, _lib.OPT_DUNE_SCREEN_TABLE, int(self.dune_screen_table)))
            _lib.check(lib.nb_pan_set_option(handle, _lib.OPT_DUNE_KERNEL, int(self.dune_kernel)))
            _lib.check(lib.nb_pan_set_option(handle, _lib.OPT_DUNE_SCREEN_MMA, int(self.dune_screen_mma)))
            _lib.check(lib.nb_pan_set_option(handle, _lib.OPT_DUNE_SKIP_T0, int(self.dune_skip_t0)))
        _lib.check(lib.nb_pan_set_option(handle, _lib.OPT_OVERLAP, int(self.overlap)))
        _lib.check(lib.nb_pan_set_option(handle, _lib.OPT_NRMP_WARM, int(self.nrmp_warm)))
        self._sent = (self.nrmp_layer.version, int(self.iter_num), float(self.iter_threshold))
        return lib

    def _push_settings(self, lib):
        cur = (self.nrmp_layer.version, int(self.iter_num), float(self.iter_threshold))
        if cur == self._sent:
            return
        nl = self.nrmp_layer
        q = (C.c_float * 3)(*[float(v) for v in nl.q_vector()])
        _lib.check(lib.nb_pan_set_adjust(self._handle, C.byref(q), float(nl.p_u.detach()), float(nl.eta.detach()),
                                         float(nl.d_max.detach()), float(nl.d_min.detach())))
        _lib.check(lib.nb_pan_set_iteration(self._handle, int(self.iter_num), float(self.iter_threshold)))
        self._sent = cur

    def close(self):
        if self._handle is not None:
            _lib.load().nb_pan_destroy(self._handle)
            self._handle = None
            self._differentiable = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset_state(self):
        """Forget the stop criterion's memory (PAN.current_nom_values, pan.py:100-105)."""
        if self._handle is not None:
            with torch.cuda.device(self.device):
                stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
                _lib.check(_lib.load().nb_pan_reset_state_async(self._handle, stream))

    def reset_envs(self, mask):
        """Forget the stop criterion's memory of the environments where ``mask`` ((B,) int32 on the device) is non-zero
        (nb_pan_reset_envs_async on the current stream, no host synchronisation); before the native handle exists there is none."""
        if self._handle is not None:
            mask = mask.to(device=self.device, dtype=torch.int32).contiguous()
            with torch.cuda.device(self.device):
                stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
                _lib.check(_lib.load().nb_pan_reset_envs_async(self._handle, int(mask.numel()), C.c_void_p(mask.data_ptr()), stream))

    # ------------------------------------------------------------------ forward
    def forward(self, nom_s: torch.Tensor, nom_u: torch.Tensor, ref_s: torch.Tensor, ref_us: torch.Tensor,
                obs_points: torch.Tensor = None, point_velocities: torch.Tensor = None, num_points: torch.Tensor = None, device_out: bool = False):
        """pan.py:109-147.  Shapes (3,T+1),(2,T),(3,T+1),(T,),(2,N),(2,N) or the same with a leading
        B.  ``num_points`` (B,) int32 marks ragged batches (extension).  Returns tensors on the
        device of ``nom_s`` with the same batching.  ``device_out=True`` with CPU (ideally pinned) inputs: the results stay on the GPU
        and the call is asynchronous (``nb_pan_forward_h2d``: chunked upload overlapped with the first DUNE pass) -- what a
        caller wants that exchanges results between GPUs before they travel back (``parallel.ShardedPAN``)."""
        batched = nom_s.dim() == 3
        un = (lambda t: t) if batched else (lambda t: None if t is None else t.unsqueeze(0))
        nom_s, nom_u, ref_s, ref_us = un(nom_s), un(nom_u), un(ref_s), un(ref_us)
        obs_points, point_velocities = un(obs_points), un(point_velocities)
        B, T = nom_s.shape[0], self.T
        assert nom_s.shape[1:] == (3, T + 1) and nom_u.shape[1:] == (2, T) and ref_s.shape[1:] == (3, T + 1)
        ref_us = ref_us.reshape(B, T)
        use_points = obs_points is not None and not self.no_obs and obs_points.shape[-1] > 0
        if not use_points:
            obs_points = point_velocities = None
        elif obs_points.shape[-1] > self.dune_max_num:  # pan.py:171-174
            self.print_once(f"down sample the obs points from {obs_points.shape[-1]} to {self.dune_max_num}")
            if num_points is None:
                idx = torch.from_numpy(decimation_indices(obs_points.shape[-1], self.dune_max_num)).to(obs_points.device)
                obs_points = obs_points.index_select(-1, idx)
                point_velocities = None if point_velocities is None else point_velocities.index_select(-1, idx)
            else:
                # ragged batch: the reference decimates each environment's OWN n_b points (an unbatched call sees (2, n_b)),
                # so the column pick is np.linspace(0, n_b-1, m).astype(int) per environment; envs with n_b <= m keep theirs
                m = self.dune_max_num
                nb = num_points.detach().to(device=obs_points.device, dtype=torch.int64).clamp(min=0, max=obs_points.shape[-1])
                step = (nb - 1).to(torch.float64) / float(m - 1) if m > 1 else torch.zeros_like(nb, dtype=torch.float64)
                idx = (torch.arange(m, device=obs_points.device, dtype=torch.float64)[None, :] * step[:, None]).to(torch.int64)  # numpy: arange * step, truncated
                idx[:, -1] = nb - 1  # linspace pins its last sample to the stop value
                keep = torch.arange(m, device=obs_points.device)[None, :].expand(B, m)
                idx = torch.where((nb > m)[:, None], idx, keep).clamp_(min=0)
                gidx = idx[:, None, :].expand(B, 2, m)
                obs_points = obs_points.gather(-1, gidx)
                point_velocities = None if point_velocities is None else point_velocities.gather(-1, gidx)
                num_points = torch.minimum(nb, torch.full_like(nb, m)).to(torch.int32)
        N = obs_points.shape[-1] if use_points else 0
        lib = self._ensure_handle(B, N)
        self._push_settings(lib)

        host_in = nom_s.device.type != "cuda"
        host = host_in and not device_out  # results on the host (synchronous call)
        in_dev = torch.device("cpu") if host_in else self.device
        io_dev = torch.device("cpu") if host else self.device
        prep = lambda t: None if t is None else t.detach().to(device=in_dev, dtype=torch.float32).contiguous()
        nom_s, nom_u, ref_s, ref_us = prep(nom_s), prep(nom_u), prep(ref_s), prep(ref_us)
        obs_points, point_velocities = prep(obs_points), prep(point_velocities)
        if num_points is not None:
            num_points = num_points.detach().to(device=in_dev, dtype=torch.int32).contiguous()
        mk = lambda *shape, dtype=torch.float32: torch.empty(shape, dtype=dtype, device=io_dev, pin_memory=host and torch.cuda.is_available())
        out_md, out_it, out_st = mk(B), mk(B, dtype=torch.int32), mk(B, dtype=torch.int32)
        # differentiable mode (LON): any adjust parameter that requires grad while autograd is recording
        leaves = self.nrmp_layer.adjust_parameters
        want_grad = torch.is_grad_enabled() and any(t.requires_grad for t in leaves)
        if want_grad != self._differentiable:
            _lib.check(lib.nb_pan_set_option(self._handle, _lib.OPT_DIFFERENTIABLE, int(want_grad)))
            self._differentiable = want_grad
        self._forward_id += 1

        def run():
            out_s, out_u, out_d = mk(B, 3, T + 1), mk(B, 2, T), mk(B, T)
            with torch.cuda.device(self.device):
                stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
                fn = lib.nb_pan_forward_host if host else (lib.nb_pan_forward_h2d if host_in else lib.nb_pan_forward)
                _lib.check(fn(self._handle, B, N, _ptr(nom_s), _ptr(nom_u), _ptr(ref_s), _ptr(ref_us), _ptr(obs_points), _ptr(point_velocities),
                              _ptr(num_points), _ptr(out_s), _ptr(out_u), _ptr(out_d), _ptr(out_md), _ptr(out_it), _ptr(out_st), stream))
            return out_s, out_u, out_d

        if want_grad:
            out_s, out_u, out_d = _PanSolve.apply(self, run, ref_s, ref_us, *leaves)
        else:
            out_s, out_u, out_d = run()
        self._last = dict(B=B, N=N, batched=batched, min_distance=out_md, iters=out_it, status=out_st, points=obs_points, use_points=use_points)
        if self.dune_layer is not None:
            if use_points:
                self.dune_layer.obstacle_points = obs_points if batched else obs_points[0]  # dune.py:76
                self.dune_layer.min_distance = out_md if batched else out_md[0]
            self.nrmp_layer.obstacle_points = None  # filled lazily by the nrmp_points property
        nom_d = None if self.no_obs else out_d.unsqueeze(1)  # (B,1,T) like the reference's (1,T)
        if batched:
            return out_s, out_u, nom_d
        return out_s[0], out_u[0], (None if nom_d is None else nom_d[0])

    # ------------------------------------------------------------------ state / properties
    @property
    def iterations(self):
        """Iterations executed per environment in the last forward (int32 tensor)."""
        return None if self._last is None else self._last["iters"]

    @property
    def status(self):
        """Per-environment solver status bits of the last forward (0 = ok)."""
        return None if self._last is None else self._last["status"]

    @property
    def ipm_iterations(self):
        """Interior point iterations of the last NRMP solve per environment (diagnostics)."""
        if self._last is None:
            return None
        out = torch.empty(self._last["B"], dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            _lib.check(_lib.load().nb_pan_read_diagnostics(self._handle, self._last["B"], _ptr(out), stream))
        return out

    def screen_stats(self, reset=True):
        """Screening statistics (dune_kernel = 4) since the last reset: dict(max_error_ratio, exact_items, candidates, screened_items,
        coarse_survivors, coarse_fallback_items).  The last two count the two-level table path of the one-warp-per-item screen: the
        points that survived its coarse bounds, and the items that took the one-level path instead (a point outside the table, or too
        many survivors)."""
        if self._handle is None or self.no_obs:
            return None
        r, c, k = (C.c_float * 3)(), (C.c_int32 * 3)(), (C.c_int32 * 2)()
        lib = _lib.load()
        _lib.check(lib.nb_pan_read_screen_stats(self._handle, C.byref(r), C.byref(c), int(reset)))
        _lib.check(lib.nb_pan_read_screen_coarse(self._handle, C.byref(k), int(reset)))
        return dict(max_error_ratio=float(r[0]), c_mu=float(r[1]), calibration_ratio=float(r[2]), exact_items=int(c[0]), candidates=int(c[1]), screened_items=int(c[2]),
                    coarse_survivors=int(k[0]), coarse_fallback_items=int(k[1]))

    def screen_table(self):
        """The screen's distance table: dict(h, half, bytes, build_ms, max_error_ratio); all zero while none is built."""
        if self._handle is None or self.no_obs:
            return None
        r = (C.c_float * 5)()
        _lib.check(_lib.load().nb_pan_read_screen_table(self._handle, C.byref(r)))
        return dict(h=float(r[0]), half=float(r[1]), bytes=int(r[2]), build_ms=float(r[3]), max_error_ratio=float(r[4]))

    def read_selection(self):
        """The M closest points per (env, step) of the last executed iteration, ascending distance:
        dict(mu (B,T+1,M,E), lam (B,T+1,M,2), points (B,T+1,M,2), distance (B,T+1,M), count (B))."""
        if self._last is None or self.no_obs:
            return None
        B, T1, M, E = self._last["B"], self.T + 1, self.nrmp_max_num, self.dune_layer.edge_dim
        mk = lambda *s, dtype=torch.float32: torch.empty(s, dtype=dtype, device=self.device)
        out = dict(mu=mk(B, T1, M, E), lam=mk(B, T1, M, 2), points=mk(B, T1, M, 2), distance=mk(B, T1, M), count=mk(B, dtype=torch.int32))
        with torch.cuda.device(self.device):
            stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            _lib.check(_lib.load().nb_pan_read_selection(self._handle, B, _ptr(out["mu"]), _ptr(out["lam"]), _ptr(out["points"]),
                                                         _ptr(out["distance"]), _ptr(out["count"]), stream))
        return out

    @property
    def min_distance(self):  # pan.py:245-252
        if self.dune_layer is None or self.no_obs:
            return inf
        return self.dune_layer.min_distance

    @property
    def dune_points(self):  # pan.py:254-260
        if self.dune_layer is None or self.no_obs:
            return None
        return tensor_to_np(self.dune_layer.points)

    @property
    def nrmp_points(self):  # pan.py:262-268, nrmp.py:135-138: closest <= M points at step 0, (2, n)
        if self.nrmp_layer is None or self.no_obs or self._last is None or not self._last["use_points"]:
            return None
        sel = self.read_selection()
        cnt = sel["count"].cpu().numpy()
        pts = sel["points"][:, 0].cpu().numpy()  # (B,M,2)
        per_env = [pts[b, :cnt[b]].T.copy() for b in range(pts.shape[0])]
        self.nrmp_layer.obstacle_points = per_env if self._last["batched"] else torch.from_numpy(per_env[0])
        return per_env if self._last["batched"] else per_env[0]

    def print_once(self, message):
        if not self.printed:
            print(message)
            self.printed = True
