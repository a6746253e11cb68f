"""The batched world's float64 oracle (oracle/world.py) against its recorded runs (tests/golden/world_oracle.npz, written by
tests/golden/make_golden_world_oracle.py): circles, convex polygons, outlines, reactive obstacles and fleets of 2 and 5 robots, for
the diff, acker and omni robots, every scan and step output and the state after every step, bit for bit.  Also: without fleet rows
the oracle is the fleet of one given by the env rows (no device needed)."""
import importlib.util
import os

import numpy as np
import pytest

from neupan_b200.world import pack_behaviors, pack_fleet, pack_scenes_ex
from oracle.world import OracleWorld

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
_spec = importlib.util.spec_from_file_location("make_golden_world_oracle", os.path.join(GOLDEN, "make_golden_world_oracle.py"))
gen = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gen)


@pytest.fixture(scope="module")
def golden():
    with np.load(os.path.join(GOLDEN, "world_oracle.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("case", list(gen.CASES))
def test_oracle_reproduces_the_recorded_run(golden, case):
    got = gen.run_case(case)
    want = {k.split("/", 1)[1]: v for k, v in golden.items() if k.startswith(case + "/")}
    assert set(want) <= set(got) and {"ranges", "collided", "states", "obs"} <= set(want)
    for a, v in want.items():
        assert np.array_equal(got[a], v), (case, a)


@pytest.mark.parametrize("case", ["rvo_mixed_acker", "outline_omni"])
def test_without_fleet_rows_the_env_rows_are_a_fleet_of_one(case):
    kind, kin, K, build = gen.CASES[case]
    rb = gen.Robot(10, 0.1, **gen.ROBOT_KW[kin])
    scenes = build(rb)
    cfg, packed, beh = gen._oracle_cfg(rb, gen.LIDAR), pack_scenes_ex(scenes), pack_behaviors(scenes)
    a = OracleWorld(cfg, packed, beh, 3)
    b = OracleWorld(cfg, packed, beh, 3, fleet=pack_fleet(scenes), K=1)
    rng = np.random.default_rng(4)
    for _ in range(20):
        act = gen._actions(rng, kin, gen.B)
        assert all(np.array_equal(x, y) for x, y in zip(a.scan(), b.scan()))
        assert all(np.array_equal(x, y) for x, y in zip(a.step(act), b.step(act)))
        for attr in ("states", "obs", "goal", "draws", "margins", "fvel", "robot_clear"):
            assert np.array_equal(getattr(a, attr), getattr(b, attr)), attr
