"""ctypes binding of libneupan_b200.so (the C ABI declared in include/neupan_b200.h).

This is the only way the Python layer reaches the CUDA kernels.  There is no CPU fallback:
if the library is missing or no CUDA device is usable the calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
# NEUPAN_B200_LIB: developer override (A/B runs of two builds of the same library)
LIB_PATH = os.environ.get("NEUPAN_B200_LIB") or os.path.join(HERE, "lib", "libneupan_b200.so")

NB_KIN = {"diff": 0, "acker": 1, "omni": 2}
NB_OK, NB_ERR_INVALID, NB_ERR_CUDA, NB_ERR_CAPACITY, NB_ERR_NO_DEVICE = 0, -1, -2, -3, -4
STATUS_MAXITER, STATUS_NUMERIC, STATUS_INFEASIBLE = 1, 2, 4
OPT_DUNE_KERNEL = 1
OPT_OVERLAP = 2
OPT_NRMP_WARM = 3
OPT_DIFFERENTIABLE = 4
OPT_DUNE_SCREEN_MMA = 5
OPT_DUNE_SKIP_T0 = 6
OPT_DUNE_SCREEN_TABLE = 7


class PanConfig(C.Structure):
    """struct nb_pan_config (include/neupan_b200.h)."""
    _fields_ = [
        ("receding", C.c_int32), ("kinematics", C.c_int32), ("edge_dim", C.c_int32), ("iter_num", C.c_int32),
        ("nrmp_max_num", C.c_int32), ("max_envs", C.c_int32), ("max_points", C.c_int32), ("device", C.c_int32),
        ("iter_threshold", C.c_float),
        ("step_time", C.c_double), ("wheelbase", C.c_double), ("max_speed", C.c_double * 2), ("max_acce", C.c_double * 2),
        ("ro_obs", C.c_double), ("bk", C.c_double),
        ("q_s", C.c_float * 3), ("p_u", C.c_float), ("eta", C.c_float), ("d_max", C.c_float), ("d_min", C.c_float),
    ]


class ScanConfig(C.Structure):
    """struct nb_scan_config (include/neupan_b200.h)."""
    _fields_ = [
        ("angle_min", C.c_double), ("angle_max", C.c_double), ("range_min", C.c_double), ("range_max", C.c_double),
        ("scan_offset", C.c_double * 3), ("angle_range", C.c_double * 2),
        ("down_sample", C.c_int32), ("velocity_mode", C.c_int32),
    ]


class IpathConfig(C.Structure):
    """struct nb_ipath_config (include/neupan_b200.h)."""
    _fields_ = [
        ("receding", C.c_int32), ("kinematics", C.c_int32), ("loop", C.c_int32), ("ind_range", C.c_int32),
        ("arrive_index_threshold", C.c_int32), ("max_envs", C.c_int32), ("device", C.c_int32), ("reserved_", C.c_int32),
        ("step_time", C.c_double), ("wheelbase", C.c_double), ("arrive_threshold", C.c_double), ("close_threshold", C.c_double),
    ]


class WorldConfig(C.Structure):
    """struct nb_world_config (include/neupan_b200.h)."""
    _fields_ = [
        ("kinematics", C.c_int32), ("num_beams", C.c_int32), ("max_envs", C.c_int32), ("device", C.c_int32),
        ("robot_num_vertices", C.c_int32), ("reserved_", C.c_int32),
        ("step_time", C.c_double), ("wheelbase", C.c_double), ("angle_min", C.c_double), ("angle_max", C.c_double),
        ("range_max", C.c_double), ("scan_offset", C.c_double * 3), ("robot_vertices", C.c_double * 16),
    ]


class WorldRobotType(C.Structure):
    """struct nb_world_robot_type (include/neupan_b200.h)."""
    _fields_ = [("kinematics", C.c_int32), ("num_vertices", C.c_int32), ("wheelbase", C.c_double), ("vertices", C.c_double * 16)]


class WorldMap(C.Structure):
    """struct nb_world_map (include/neupan_b200.h)."""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("origin", C.c_double * 2), ("resolution", C.c_double)]


class WorldActuation(C.Structure):
    """struct nb_world_actuation (include/neupan_b200.h)."""
    _fields_ = [("vel_min", C.c_double * 2), ("vel_max", C.c_double * 2), ("acce", C.c_double * 2), ("alpha", C.c_double * 4)]


_FP = C.c_void_p  # device or host float* / int32*: passed as raw addresses

# name -> (restype, argtypes); every symbol include/neupan_b200.h declares
SYMBOLS = {
    "nb_weight_count": (C.c_int64, [C.c_int32]),
    "nb_pan_create": (C.c_int, [C.POINTER(PanConfig), _FP, C.c_int64, _FP, _FP, C.POINTER(C.c_void_p)]),
    "nb_pan_destroy": (C.c_int, [C.c_void_p]),
    "nb_pan_forward": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32] + [_FP] * 13 + [C.c_void_p]),
    "nb_pan_forward_host": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32] + [_FP] * 13 + [C.c_void_p]),
    "nb_pan_forward_h2d": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32] + [_FP] * 13 + [C.c_void_p]),
    "nb_pan_set_adjust": (C.c_int, [C.c_void_p, C.POINTER(C.c_float * 3), C.c_float, C.c_float, C.c_float, C.c_float]),
    "nb_pan_set_iteration": (C.c_int, [C.c_void_p, C.c_int32, C.c_float]),
    "nb_pan_set_option": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32]),
    "nb_pan_reset_state": (C.c_int, [C.c_void_p]),
    "nb_pan_reset_state_async": (C.c_int, [C.c_void_p, C.c_void_p]),
    "nb_pan_reset_envs_async": (C.c_int, [C.c_void_p, C.c_int32, _FP, C.c_void_p]),
    "nb_pan_backward": (C.c_int, [C.c_void_p, C.c_int32] + [_FP] * 6 + [C.c_void_p]),
    "nb_pan_read_selection": (C.c_int, [C.c_void_p, C.c_int32] + [_FP] * 5 + [C.c_void_p]),
    "nb_pan_read_screen_stats": (C.c_int, [C.c_void_p, C.POINTER(C.c_float * 3), C.POINTER(C.c_int32 * 3), C.c_int32]),
    "nb_pan_read_screen_table": (C.c_int, [C.c_void_p, C.POINTER(C.c_float * 5)]),
    "nb_pan_read_screen_coarse": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32 * 2), C.c_int32]),
    "nb_pan_read_diagnostics": (C.c_int, [C.c_void_p, C.c_int32, _FP, C.c_void_p]),
    "nb_dune_forward": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32] + [_FP] * 5 + [C.c_void_p]),
    "nb_nrmp_forward": (C.c_int, [C.c_void_p, C.c_int32] + [_FP] * 10 + [C.c_void_p]),
    "nb_scan_to_points": (C.c_int, [C.c_int32, C.c_int32, _FP, _FP, _FP, C.POINTER(ScanConfig), C.c_int32, _FP, _FP, _FP, C.c_void_p]),
    "nb_ipath_create": (C.c_int, [C.POINTER(IpathConfig), C.POINTER(C.c_void_p)]),
    "nb_ipath_destroy": (C.c_int, [C.c_void_p]),
    "nb_ipath_set_paths": (C.c_int, [C.c_void_p, C.c_int32, _FP, C.c_int64, _FP, C.c_int32, _FP, _FP]),
    "nb_ipath_step": (C.c_int, [C.c_void_p, C.c_int32, _FP, _FP, C.c_double, _FP, _FP, _FP, _FP, _FP, C.c_void_p]),
    "nb_ipath_step_ex": (C.c_int, [C.c_void_p, C.c_int32, _FP, _FP, _FP, C.c_double, _FP, _FP, _FP, _FP, _FP, C.c_void_p]),
    "nb_ipath_reset": (C.c_int, [C.c_void_p]),
    "nb_ipath_reset_async": (C.c_int, [C.c_void_p, C.c_void_p]),
    "nb_ipath_read_state": (C.c_int, [C.c_void_p, C.c_int32, _FP, _FP, _FP, _FP, C.c_void_p]),
    "nb_world_create": (C.c_int, [C.POINTER(WorldConfig), C.POINTER(C.c_void_p)]),
    "nb_world_destroy": (C.c_int, [C.c_void_p]),
    "nb_world_check_scenes": (C.c_int, [C.POINTER(WorldConfig), C.c_int32, _FP, _FP, _FP, _FP, _FP]),
    "nb_world_set_scenes": (C.c_int, [C.c_void_p, C.c_int32, _FP, _FP, _FP, _FP, _FP]),
    "nb_world_check_scenes_ex": (C.c_int, [C.POINTER(WorldConfig), C.c_int32, _FP, _FP, _FP, _FP, _FP, _FP]),
    "nb_world_set_scenes_ex": (C.c_int, [C.c_void_p, C.c_int32, _FP, _FP, _FP, _FP, _FP, _FP]),
    "nb_world_scan": (C.c_int, [C.c_void_p, C.c_int32, _FP, _FP, _FP, C.c_void_p]),
    "nb_world_step": (C.c_int, [C.c_void_p, C.c_int32, _FP, _FP, _FP, _FP, C.c_void_p]),
    "nb_world_read_state": (C.c_int, [C.c_void_p, C.c_int32, _FP, _FP, _FP, _FP, C.c_void_p]),
    "nb_world_check_behaviors": (C.c_int, [C.POINTER(WorldConfig), C.c_int32] + [_FP] * 7 + [C.c_uint64]),
    "nb_world_set_behaviors": (C.c_int, [C.c_void_p, C.c_int32, _FP, C.c_uint64]),
    "nb_world_read_behaviors": (C.c_int, [C.c_void_p, C.c_int32, _FP, _FP, C.c_void_p]),
    "nb_world_check_fleet": (C.c_int, [C.POINTER(WorldConfig), C.c_int32, C.c_int32, _FP]),
    "nb_world_set_fleet": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, _FP]),
    "nb_world_check_fleet_ex": (C.c_int, [C.POINTER(WorldConfig), C.c_int32, _FP, C.c_int32, C.c_int32, _FP, _FP]),
    "nb_world_set_fleet_ex": (C.c_int, [C.c_void_p, C.c_int32, _FP, C.c_int32, C.c_int32, _FP, _FP]),
    "nb_world_check_maps": (C.c_int, [C.POINTER(WorldConfig), C.c_int32, _FP, C.c_int32, C.c_int32, _FP, _FP, C.c_int32, _FP, _FP, _FP,
                                      C.c_double]),
    "nb_world_set_maps": (C.c_int, [C.c_void_p, C.c_int32, _FP, _FP, _FP, C.c_double]),
    "nb_world_check_map_contact": (C.c_int, [C.POINTER(WorldConfig), C.c_int32] + [_FP] * 7 + [C.c_int32, _FP, _FP, _FP, _FP]),
    "nb_world_set_map_contact": (C.c_int, [C.c_void_p, C.c_int32, _FP]),
    "nb_world_read_map_contact": (C.c_int, [C.c_void_p, C.c_int32, _FP, C.c_void_p]),
    "nb_world_check_obstacle_contact": (C.c_int, [C.POINTER(WorldConfig), C.c_int32] + [_FP] * 8),
    "nb_world_set_obstacle_contact": (C.c_int, [C.c_void_p, C.c_int32, _FP]),
    "nb_world_read_obstacle_contact": (C.c_int, [C.c_void_p, C.c_int32, _FP, C.c_void_p]),
    "nb_world_check_episodes": (C.c_int, [C.POINTER(WorldConfig), C.c_int32, C.c_int32, _FP, C.c_int32, C.c_int32]),
    "nb_world_set_episodes": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32]),
    "nb_world_read_episodes": (C.c_int, [C.c_void_p, C.c_int32] + [_FP] * 10 + [C.c_void_p]),
    "nb_world_set_actuation": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(WorldActuation), C.c_uint64]),
    "nb_world_set_lidar_noise": (C.c_int, [C.c_void_p, C.c_double, C.c_double, C.c_uint64]),
    "nb_world_read_commands": (C.c_int, [C.c_void_p, C.c_int32, _FP, C.c_void_p]),
    "nb_dune_labels": (C.c_int, [C.c_int32, _FP, _FP, C.c_int64, _FP, _FP, _FP, _FP, C.c_void_p]),
    "nb_dune_train_create": (C.c_int, [C.c_int32, _FP, _FP, _FP, C.c_int64, C.c_int32, C.POINTER(C.c_void_p)]),
    "nb_dune_train_destroy": (C.c_int, [C.c_void_p]),
    "nb_dune_train_epoch": (C.c_int, [C.c_void_p, _FP, _FP, _FP, C.c_int64, C.c_int32, _FP, C.c_float, C.c_int32, _FP, C.c_void_p]),
    "nb_dune_train_get_weights": (C.c_int, [C.c_void_p, _FP]),
    "nb_launch_count": (C.c_int64, []),
    "nb_buffer_count": (C.c_int64, []),
    "nb_last_error": (C.c_char_p, []),
    "nb_version": (C.c_int, []),
}

_lib = None


def load() -> C.CDLL:
    """Loads the shared library (built by ``python -m neupan_b200.build``); raises if absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -m neupan_b200.build` "
                "(neupan_b200 has no CPU fallback; the CUDA library is the product)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(lib, name)  # AttributeError if the .so does not export it
            fn.restype, fn.argtypes = res, args
        _lib = lib
    return _lib


class NeupanB200Error(RuntimeError):
    pass


def check(rc: int):
    if rc == NB_OK:
        return
    msg = load().nb_last_error().decode()
    if rc == NB_ERR_INVALID:
        raise ValueError(msg)
    if rc == NB_ERR_CAPACITY:
        raise ValueError("capacity exceeded: " + msg)
    raise NeupanB200Error(msg)


def unpack_weights(flat: np.ndarray, reference_state_dict) -> dict:
    """Inverse of pack_weights: a flat float32 vector -> {key: tensor} with the shapes of `reference_state_dict`."""
    import torch

    out, off = {}, 0
    for idx in (0, 1, 3, 5, 6, 8, 10, 11, 13):
        for kind in ("weight", "bias"):
            key = f"MLP.{idx}.{kind}"
            shape = tuple(reference_state_dict[key].shape)
            n = int(np.prod(shape))
            out[key] = torch.from_numpy(np.array(flat[off:off + n], dtype=np.float32).reshape(shape))
            off += n
    assert off == flat.size
    return out


def pack_weights(state_dict) -> np.ndarray:
    """Concatenates an ObsPointNet state_dict (keys MLP.{0,1,3,5,6,8,10,11,13}.{weight,bias},
    neupan/blocks/obs_point_net.py:31-46) into the flat float32 layout nb_pan_create expects."""
    parts = []
    for idx in (0, 1, 3, 5, 6, 8, 10, 11, 13):
        for kind in ("weight", "bias"):
            v = state_dict[f"MLP.{idx}.{kind}"]
            v = v.detach().cpu().numpy() if hasattr(v, "detach") else np.asarray(v)
            parts.append(np.ascontiguousarray(v, dtype=np.float32).reshape(-1))
    return np.concatenate(parts)
