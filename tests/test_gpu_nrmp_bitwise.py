"""The compile-time NRMP specialisations (C4 shape T = 10, M = 10 and C5 shape T = 15, M = 10) reproduce golden outputs bit for
bit: S, U, D, status and interior point iterations of tests/golden/nrmp_bitwise.npz (make_golden_nrmp_bitwise.py), for the diff,
acker and omni robots under the shipped bounds and three bound regimes.  Their addressing and loop shapes are free to change; the
floating-point operations and their order are not."""
import importlib.util
import os

import numpy as np
import pytest

from test_gpu_nrmp_shapes import _solve
from test_oracle_nrmp_shapes import case_config

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("make_golden_nrmp_bitwise", os.path.join(HERE, "golden", "make_golden_nrmp_bitwise.py"))
gen = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gen)
ENVS, INPUTS, OUTPUTS, case_name = gen.ENVS, gen.INPUTS, gen.OUTPUTS, gen.case_name

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(HERE, "golden", "nrmp_bitwise.npz")
CASES = list(gen.cases())


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("T,M,kin,regime", CASES, ids=[case_name(*c) for c in CASES])
def test_specialisation_reproduces_golden_bits(golden, T, M, kin, regime):
    name = case_name(T, M, kin, regime)
    inp = {k: golden[f"{name}.{k}"] for k in INPUTS}
    assert inp["nom_s"].shape[0] == ENVS
    cfg = case_config(kin, T, M, regime)
    out = _solve(cfg, dict(inp, points=None, velocities=None), inp["fa"], inp["fb"])
    for k in OUTPUTS:
        want = golden[f"{name}.{k}"]
        assert out[k].dtype == want.dtype and np.array_equal(out[k], want), (name, k, np.argwhere(out[k] != want)[:5].tolist())
