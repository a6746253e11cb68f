"""Pins the NRMP convex program to the REFERENCE'S OWN CODE.

``oracle/cvx_shim.py`` stands in for cvxpy / cvxpylayers, so ``neupan/blocks/nrmp.py:263-383`` and
``neupan/robot/robot.py:73-236`` execute unmodified and produce the program as arrays.  What the reference's code built and
returned is stored in ``tests/golden/ref_program.npz`` (``tests/golden/make_golden_refprog.py``).  Checked here, for
diff / acker / omni, scalar and vector q_s, with and without obstacle rows:

* the reference's objective equals ``oracle.nrmp.objective`` at random points (feasible or not);
* the oracle's optimum (float64 interior point, ``oracle/ipm.py``) satisfies the reference's constraints and passes a
  solver-free KKT certificate *of the reference's program*;
* the reference's own ``NRMP.forward`` (shim solver: HiGHS + active-set polish) returns the same trajectory;
* the reference's whole ``PAN.forward`` (its torch DUNE code + its NRMP through the shim) agrees with ``oracle.pan.OraclePAN``.

Where the reference checkout is present, the fixtures are also checked to be current.  What stays unobservable: ECOS' own output.
"""
import importlib.util
import os

import numpy as np
import pytest

from helpers import oracle_factory, robot_spec
from oracle import dune as od, ipm as oipm, nrmp as onr, refload
from oracle.cvx_shim import Canonical

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("make_golden_refprog", os.path.join(HERE, "golden", "make_golden_refprog.py"))
mgr = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mgr)
GOLD = np.load(os.path.join(HERE, "golden", "ref_program.npz"))
CASES = mgr.CASES


def _problem_and_reference(cname, adjust_over, M):
    """The oracle's program of a case (no reference code involved) and, from the fixtures, the reference's canonical program of
    the same case, the solution its NRMP.forward found (float64) and its S, U, D."""
    i = CASES.index((cname, adjust_over, M))
    cfg, adjust, Mv, inp = mgr.case_inputs(cname, adjust_over, M)
    if Mv > 0:
        mu, lam, sp, h, spec = mgr.dune_lists(cfg, inp)
        fa, fb = od.nrmp_coefficients(h, mu, lam, sp, cfg.T, Mv)
        fa, fb = fa.numpy(), fb.numpy()
    else:
        _, spec = robot_spec(cfg)
        fa = fb = None
    prob = onr.build_problem(spec, onr.Adjust(**adjust), inp["nom_s"][0], inp["nom_u"][0], inp["ref_s"][0], inp["ref_us"][0], fa, fb, Mv)
    p = f"case{i}"
    ref = (GOLD[f"{p}.S"], GOLD[f"{p}.U"], GOLD[f"{p}.D"] if f"{p}.D" in GOLD.files else None)
    return cfg, prob, Canonical.from_arrays(GOLD, p), GOLD[f"{p}.x_ref"], ref


def _stack_x(prob, S, U, D):
    parts = [np.asarray(S, float).reshape(-1), np.asarray(U, float).reshape(-1)]
    if prob.M > 0:
        parts.append(np.asarray(D, float).reshape(-1))
    return np.concatenate(parts)


@pytest.mark.parametrize("cname,adjust,M", CASES)
def test_reference_objective_equals_oracle_objective(cname, adjust, M):
    _, prob, can, _, _ = _problem_and_reference(cname, adjust, M)
    rng = np.random.default_rng(5)
    for _ in range(6):
        S = prob.nom_s + rng.normal(0, 0.5, prob.nom_s.shape)
        U = rng.normal(0, 2.0, (2, prob.T))
        D = rng.uniform(-0.5, 1.5, (1, prob.T))
        a, b = can.objective(_stack_x(prob, S, U, D)), onr.objective(prob, S, U, D[0])
        assert abs(a - b) <= 1e-9 * max(1.0, abs(b)), (a, b)


@pytest.mark.parametrize("cname,adjust,M", CASES)
def test_oracle_optimum_is_optimal_for_the_reference_program(cname, adjust, M):
    _, prob, can, xr, (Sr, Ur, Dr) = _problem_and_reference(cname, adjust, M)
    S, U, D, _ = oipm.solve_ipm(prob)
    x = _stack_x(prob, S, U, D)
    res, viol = can.kkt_certificate(x, act_tol=1e-7)
    scale = max(1.0, float(np.abs(can.gradient(x)).max()))
    assert viol < 1e-8, viol  # the reference's constraints hold at the oracle's optimum
    assert res < 2e-6 * scale, (res, scale)  # and its gradient is a combination of active normals
    # the reference's own forward (shim solver) lands on the same point; xr is float64, before the reference's cast to float32
    assert can.violation(xr) < 1e-8
    assert can.objective(x) <= can.objective(xr) + 1e-8 * max(1.0, abs(can.objective(xr)))
    assert np.abs(U - Ur).max() < 2e-5 and np.abs(S - Sr).max() < 2e-5
    if prob.M > 0:
        assert np.abs(D - Dr).max() < 2e-5


def test_reference_parameter_values_equal_oracle_parameters():
    """generate_parameter_value of the reference (nrmp.py:152-166, robot.py:239-316) vs oracle.nrmp.build_problem: bit for bit."""
    for cname in mgr.PARAM_CONFIGS:
        cfg, prob, _, _, _ = _problem_and_reference(cname, {}, None)
        T = cfg.T
        vals = [GOLD[f"params_{cname}.{k}"] for k in range(3 + 5 * T)]
        assert np.array_equal(vals[0], prob.nom_s.astype(np.float32))
        assert np.array_equal(vals[1], prob.gamma_a.astype(np.float32))
        assert np.array_equal(vals[2], prob.gamma_b.astype(np.float32))
        for k in range(T):
            assert np.array_equal(vals[3 + k], prob.A[k].astype(np.float32))
            assert np.array_equal(vals[3 + T + k], prob.B[k].astype(np.float32))
            assert np.array_equal(vals[3 + 2 * T + k].reshape(-1), prob.C[k].astype(np.float32))
            assert np.array_equal(vals[3 + 3 * T + k], prob.fa[k].astype(np.float32))
            assert np.array_equal(vals[3 + 4 * T + k].reshape(-1), prob.fb[k].astype(np.float32))


@pytest.mark.parametrize("cname,K", mgr.PAN_RUNS)
def test_reference_pan_forward_equals_oracle_pan(cname, K):
    """The reference's PAN.forward end to end (pan.py:109-147) with only the solver swapped vs OraclePAN."""
    cfg, N, inp = mgr.pan_inputs(cname)
    for b in range(mgr.PAN_ENVS):
        p = f"pan_{cname}_{K}_{b}"
        op_ = oracle_factory(cfg, K=K, N=N)()
        vel = None if inp["velocities"] is None else inp["velocities"][b]
        So, Uo, Do = op_.forward(inp["nom_s"][b], inp["nom_u"][b], inp["ref_s"][b], inp["ref_us"][b], inp["points"][b], vel)
        assert np.abs(GOLD[f"{p}.S"] - So).max() < 1e-4 and np.abs(GOLD[f"{p}.U"] - Uo).max() < 1e-4 and np.abs(GOLD[f"{p}.D"] - Do).max() < 1e-4
        assert abs(float(GOLD[f"{p}.md"]) - op_.min_distance) < 1e-6


@pytest.mark.skipif(not refload.reference_available(), reason="needs the reference checkout")
def test_program_fixtures_are_current():
    """Re-runs the reference's code for one program case, one parameter set and one PAN run: same arrays as the fixtures."""
    fresh = {**mgr.reference_case(5), **mgr.reference_params("C2"), **mgr.reference_pan("C1", 2)}
    for k, v in fresh.items():
        assert np.array_equal(np.asarray(v), GOLD[k]), k
