"""Continuous episodes in the batched world, on the CPU: every refusal of nb_world_check_episodes and of the Python bank check, and the
numpy restatement of the end test and the slot assignment (tests/world_episode_oracle.py) on hand-made end patterns (no device
needed)."""
import ctypes as C
import math

import numpy as np
import pytest

from neupan_b200 import _lib, build as nb_build
from neupan_b200.robot import robot as Robot
from neupan_b200.world import check_bank, circle_swap, dyna_obs, make_config, mixed_swap, pack_robot_types
from world_episode_oracle import EpisodeOracle

LIDAR = dict(angle_min=-math.pi, angle_max=math.pi, range_min=0.0, range_max=10.0, number=36)


@pytest.fixture(scope="module")
def lib():
    nb_build.build()
    return _lib.load()


def _cfg(max_envs=8):
    return make_config(Robot(10, 0.1, kinematics="diff", length=1.6, width=2.0), LIDAR, 0.1, max_envs)


def _check(lib, cfg, S, K, rtype, slots, max_steps):
    rt = None if rtype is None else np.ascontiguousarray(rtype, np.int32)
    return lib.nb_world_check_episodes(C.byref(cfg), S, K, None if rt is None else C.c_void_p(rt.ctypes.data), slots, max_steps)


def test_check_episodes_accepts_a_valid_bank(lib):
    cfg = _cfg()
    assert _check(lib, cfg, 8, 1, None, 3, 1) == 0
    assert _check(lib, cfg, 8, 3, [0, 1, 2] * 8, 8, 100) == 0
    assert _check(lib, cfg, 1, 16, None, 1, 1) == 0


@pytest.mark.parametrize("S, K, rtype, slots, max_steps, msg", [
    (8, 1, None, 0, 10, "slots = 0 outside [1, S = 8]"),
    (8, 1, None, 9, 10, "slots = 9 outside [1, S = 8]"),
    (8, 1, None, 4, 0, "max_steps = 0 must be >= 1"),
    (9, 1, None, 4, 10, "S = 9 scenes outside [1, max_envs = 8]"),
    (0, 1, None, 1, 10, "S = 0 scenes outside"),
    (4, 17, None, 2, 10, "K = 17 robots per scene"),
    (4, 2, [0, 1, 0, 1, 1, 1, 0, 1], 2, 10, "scene 2, robot 0: type 1 but robot 0 of scene 0 has type 0"),
    (3, 3, [0, 1, 2, 0, 1, 2, 0, 2, 2], 2, 10, "scene 2, robot 1: type 2 but robot 1 of scene 0 has type 1"),
])
def test_check_episodes_refusals(lib, S, K, rtype, slots, max_steps, msg):
    assert _check(lib, _cfg(), S, K, rtype, slots, max_steps) == _lib.NB_ERR_INVALID
    assert msg in lib.nb_last_error().decode()


def test_python_bank_check_refusals():
    scenes = dyna_obs(6)
    check_bank(scenes, 2, 10, 8)
    with pytest.raises(ValueError, match=r"slots = 7 outside \[1, S = 6\]"):
        check_bank(scenes, 7, 10, 8)
    with pytest.raises(ValueError, match=r"slots = 0 outside"):
        check_bank(scenes, 0, 10, 8)
    with pytest.raises(ValueError, match="max_steps = 0 must be >= 1"):
        check_bank(scenes, 2, 0, 8)
    with pytest.raises(ValueError, match=r"S = 6 scenes outside \[1, max_envs = 5\]"):
        check_bank(scenes, 2, 10, 5)
    mixed = circle_swap(3, robots=2) + circle_swap(1, robots=3)
    with pytest.raises(ValueError, match="scene 3 has 3 robots but scene 0 has 2"):
        check_bank(mixed, 2, 10, 8)
    swaps = mixed_swap(4, robots=3)
    check_bank(swaps, 2, 10, 8)
    swaps[2]["robots"][1] = dict(swaps[2]["robots"][1], type=0)
    with pytest.raises(ValueError, match="scene 2, robot 1: type 0 but robot 1 of scene 0 has type 1"):
        check_bank(swaps, 2, 10, 8)
    # the same bank through the C check: the packed types name the same scene and robot
    nb_build.build()
    lib = _lib.load()
    assert _check(lib, _cfg(), 4, 3, pack_robot_types(swaps), 2, 10) == _lib.NB_ERR_INVALID
    assert "scene 2, robot 1: type 0 but robot 1 of scene 0 has type 1" in lib.nb_last_error().decode()


# ---- the restatement on hand-made end patterns ----------------------------------------------------------------------------

def _pattern(ends, K=1):
    """flags(s, t): scene s ends by flags at step ends[s] (None: never), robot 0 collided for odd s, every robot arrived for even s;
    clearance 10 - t."""
    def flags(s, t):
        e = ends[s]
        hit = e is not None and t >= e
        col = np.full(K, 1 if hit and s % 2 else 0, np.int32)
        arr = np.full(K, 1 if hit and s % 2 == 0 else 0, np.int32)
        if hit and s % 2:
            col[1:] = 0
            arr[1:] = 1
        return col, arr, np.full(K, 10.0 - t, np.float32)
    return flags


def test_several_slots_end_in_the_same_step():
    o = EpisodeOracle(S=7, slots=3, K=1, max_steps=50)
    trace = o.run(_pattern([2, 2, 2, 1, 3, 1, 1]))
    assert trace[:4].tolist() == [[0, 1, 2], [0, 1, 2], [3, 4, 5], [6, 4, 5]]
    assert o.end_step.tolist() == [2, 2, 2, 1, 3, 1, 1] and (o.reason == 1).all()
    assert o.slot.tolist() == [0, 1, 2, 0, 1, 2, 0]
    assert o.finished == 7 and not o.live.any()


def test_bank_runs_out_mid_step():
    o = EpisodeOracle(S=5, slots=4, K=1, max_steps=50)
    o.advance(_pattern([1, 1, 1, 4, 1]))  # three slots end together, one scene is left: slot 0 takes it, slots 1 and 2 go idle
    assert o.scene_of.tolist() == [4, 1, 2, 3] and o.live.tolist() == [1, 0, 0, 1] and o.reset.tolist() == [1, 0, 0, 0]
    assert o.next == 7 and o.finished == 3
    before = (o.min_clearance.copy(), o.end_step.copy())
    o.advance(_pattern([1, 1, 1, 4, 1]))
    assert o.live.tolist() == [0, 0, 0, 1] and o.finished == 4
    assert np.array_equal(o.min_clearance[1:3], before[0][1:3]) and np.array_equal(o.end_step[1:3], before[1][1:3])  # idle: frozen


def test_s_not_a_multiple_of_slots_and_timeouts():
    o = EpisodeOracle(S=7, slots=3, K=2, max_steps=4)
    trace = o.run(_pattern([None, 2, None, 1, None, None, 3], K=2))
    assert o.finished == 7
    assert o.reason.tolist() == [2, 1, 2, 1, 2, 2, 1] and o.end_step.tolist() == [4, 2, 4, 1, 4, 4, 3]
    assert trace[0].tolist() == [0, 1, 2] and trace[2].tolist() == [0, 3, 2] and trace[3].tolist() == [0, 4, 2]
    assert (o.arrive_step[[0, 1, 4, 5]] == -1).all() and o.arrive_step[2:4].tolist() == [-1, 2]  # scene 1: robot 1 arrived at 2
    assert o.min_clearance[0] == np.float32(6.0)  # 10 - 4 after four steps


def test_flags_win_a_tie_with_the_timeout():
    o = EpisodeOracle(S=2, slots=1, K=1, max_steps=3)
    o.run(_pattern([3, None]))
    assert o.reason.tolist() == [1, 2] and o.end_step.tolist() == [3, 3]


def test_slots_equal_scenes_and_max_steps_one():
    o = EpisodeOracle(S=4, slots=4, K=1, max_steps=1)
    trace = o.run(_pattern([None, 1, None, None]))
    assert trace.tolist() == [[0, 1, 2, 3]]
    assert o.reason.tolist() == [2, 1, 2, 2] and (o.end_step == 1).all() and not o.live.any() and not o.reset.any()
    o = EpisodeOracle(S=5, slots=2, K=1, max_steps=1)
    trace = o.run(_pattern([None] * 5))
    assert trace.tolist() == [[0, 1], [2, 3], [4, 3]] and o.slot.tolist() == [0, 1, 0, 1, 0]
