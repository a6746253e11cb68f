"""The NRMP solve at every kernel instantiation, for the three kinematics, and under bound regimes the shipped configurations never
reach: the case tables and the problem builder of tests/test_gpu_nrmp_shapes.py, and their checks on the CPU.

launch_nrmp (csrc/nrmp.cu) sends a handle to one of nine instantiations nrmp_kernel<HPL, SMALL, TT, MM>, chosen from the
horizon T, nrmp_max_num M and TM = T M; the kinematics is a run-time branch inside every one of them.  `instantiation` mirrors
that table.  Every shape of SHAPES runs with the diff (C4), acker (C2) and omni (C5) robot, each config with its own robot and
checkpoint.  Obstacle coefficients fa / fb come from the float64 oracle's DUNE selection, so the NRMP solve is compared on its own,
without near-ties at the top-M boundary.

Checked here: the float64 interior point oracle solves every case and passes the KKT certificate, every bound regime has the
active constraint families it claims at the oracle's optimum, and the case tables reach every branch of the dispatch mirror."""
import dataclasses
from math import inf

import numpy as np
import pytest

from helpers import CONFIGS, make_inputs, robot_spec
from oracle import dune as od, ipm as oi, nrmp as onr
from test_gpu_parity import _oracle_dune

KIN_CONFIG = {"diff": "C4", "acker": "C2", "omni": "C5"}
KINS = tuple(KIN_CONFIG)

# (T, M): both sides of every switch of the dispatch table.  T = 1 has no rate rows; (16, 2): TM = 32 = 2T; (11, 3): TM = 33 and
# 2T = 22 is not a multiple of the 8-row DMMA tile; (15, 9) sits next to the (15, 10) specialisation; (8, 32): M at its largest;
# (17, 1): the first T with SMALL = false; (32, *): the largest T of the ABI
SHAPES = [(1, 8), (16, 2), (11, 3), (8, 8), (13, 5), (16, 8), (15, 9), (16, 10), (7, 24), (8, 32), (16, 16), (17, 1), (20, 6), (32, 4),
          (17, 10), (25, 7), (32, 8), (10, 10), (15, 10)]
# one shape per instantiation, for the bound regimes, the status paths and the schedule ((16, 16), not (7, 24): at T <= 8 the
# diff robot's tight speed box holds all along the horizon and its rate rows stay inactive)
REPRESENTATIVE = [(16, 2), (11, 3), (13, 5), (15, 9), (16, 16), (20, 6), (25, 7), (10, 10), (15, 10)]
ENVS = 6     # per case: half `annulus`, half `obstacles`
N_CLOUD = 64  # points per environment (>= the largest M)

FAMILIES = ("speed", "angular", "rate_speed", "rate_angular", "d_upper", "d_lower")
# bounds under which every family is active in some environment of every case, per kinematics (measured on the oracle: the
# shipped configs all allow 8 m/s against a 4 m/s reference and leave the angular rows inactive).  acker: U[1] is the steering
# angle; omni: U[1] is the heading command, around start headings in [-pi, pi]
TIGHT = {
    "diff": dict(max_speed=[2.5, 0.15], max_acce=[0.3, 0.4], d_max=0.6, d_min=0.35),
    "acker": dict(max_speed=[2.5, 0.05], max_acce=[1.0, 0.3], d_max=0.6, d_min=0.35),
    "omni": dict(max_speed=[2.5, 1.0], max_acce=[1.0, 1.0], d_max=0.6, d_min=0.35),
}
# regime -> families that must be active in at least one environment of every case
REGIMES = {
    "tight": FAMILIES,
    # the finite entries of TIGHT with the others infinite (acker: its steering box stays finite, 1.57)
    "speed_box_and_angular_rate": ("speed", "rate_angular", "d_upper"),   # max_speed = [s, inf], max_acce = [inf, a]
    "angular_box_and_speed_rate": ("angular", "rate_speed", "d_upper"),   # max_speed = [inf, s], max_acce = [a, inf]
    "d_min_negative": ("d_upper",),        # the shipped bounds with d_min = -0.2: the program uses max(d_min, 0)
    "fewer_points_than_m": ("d_upper",),   # the shipped bounds, N = M // 2: rows pn..M repeat row 0 (nrmp.py:258-259)
}


def instantiation(T, M):
    """(HPL, SMALL, TT, MM) of the nrmp_kernel that launch_nrmp (csrc/nrmp.cu) launches for horizon T and nrmp_max_num M."""
    if (T, M) == (10, 10):
        return (4, True, 10, 10)
    if (T, M) == (15, 10):
        return (5, True, 15, 10)
    hpl = (T * M + 31) // 32
    if T <= 16:
        for h in (1, 2, 4, 5):
            if hpl <= h:
                return (h, True, 0, 0)
        return (8, True, 0, 0)
    return (4 if hpl <= 4 else 8, False, 0, 0)


ALL_INSTANTIATIONS = {(1, True, 0, 0), (2, True, 0, 0), (4, True, 0, 0), (5, True, 0, 0), (8, True, 0, 0), (4, False, 0, 0), (8, False, 0, 0),
                      (4, True, 10, 10), (5, True, 15, 10)}


def label(inst):
    h, small, tt, mm = inst
    return f"nrmp_kernel<{h}, {'true' if small else 'false'}, {tt}, {mm}>"


def case_config(kin, T, M, regime=None, N=N_CLOUD, robot=None, adjust=None):
    """The base config of the kinematics at horizon T, M rows per step and N points, with the bounds of `regime`."""
    base = CONFIGS[KIN_CONFIG[kin]]
    rk, adj = dict(base.robot_kwargs), dict(base.adjust)
    tight = TIGHT[kin]
    if regime is not None and regime != "d_min_negative" and regime != "fewer_points_than_m":
        adj.update(d_max=tight["d_max"], d_min=tight["d_min"])
        s, a = tight["max_speed"], tight["max_acce"]
        rk.update({"tight": dict(max_speed=s, max_acce=a),
                   "speed_box_and_angular_rate": dict(max_speed=[s[0], inf], max_acce=[inf, a[1]]),
                   "angular_box_and_speed_rate": dict(max_speed=[inf, s[1]], max_acce=[a[0], inf])}[regime])
    if regime == "d_min_negative":
        adj["d_min"] = -0.2
    if regime == "fewer_points_than_m":
        N = max(1, M // 2)
    rk.update(robot or {}); adj.update(adjust or {})
    return dataclasses.replace(base, T=T, M=M, N=N, robot_kwargs=rk, adjust=adj)


def case_inputs(cfg, B=ENVS, env_offset=0):
    """B environments of the config: the first half in the `annulus` scene, the rest in `obstacles` (other environment indices)."""
    na = B - B // 2
    a = make_inputs(cfg, B=na, scene="annulus", env_offset=env_offset)
    o = make_inputs(cfg, B=B - na, scene="obstacles", env_offset=env_offset + na)
    return {k: None if a[k] is None else np.ascontiguousarray(np.concatenate([a[k], o[k]])) for k in a}


def build_case(cfg, inp):
    """fa (B, T, M, 2) / fb (B, T, M) from the oracle's DUNE selection (None when M = 0) and the float64 problems."""
    B, T, M = inp["nom_s"].shape[0], cfg.T, cfg.M
    rb, spec = robot_spec(cfg)
    fa = fb = None
    if M > 0:
        fa = np.zeros((B, T, M, 2), np.float32); fb = np.zeros((B, T, M), np.float32)
        for b in range(B):
            (mu, lam, sp, _, _), h = _oracle_dune(cfg, inp, b)
            a, c = od.nrmp_coefficients(h, mu, lam, sp, T, M)
            fa[b], fb[b] = a.numpy(), c.numpy()
    adj = onr.Adjust(**cfg.adjust)
    probs = [onr.build_problem(spec, adj, inp["nom_s"][b], inp["nom_u"][b], inp["ref_s"][b], inp["ref_us"][b],
                               None if fa is None else fa[b], None if fb is None else fb[b], M) for b in range(B)]
    return fa, fb, probs


def active_counts(prob, U, D, tol=1e-6):
    """Rows of each constraint family that hold with equality (slack <= tol) at (U, D)."""
    sb, ab = prob.speed_bound, prob.acce_bound
    dU = np.abs(np.diff(U, axis=1))
    D = np.zeros(0) if D is None else np.asarray(D).reshape(-1)
    return dict(speed=int(np.sum(np.abs(U[0]) >= sb[0] - tol)), angular=int(np.sum(np.abs(U[1]) >= sb[1] - tol)),
                rate_speed=int(np.sum(dU[0] >= ab[0] - tol)), rate_angular=int(np.sum(dU[1] >= ab[1] - tol)),
                d_upper=int(np.sum(D >= prob.d_max - tol)), d_lower=int(np.sum(D <= max(prob.d_min, 0.0) + tol)))


def _certified(prob):
    """The oracle's optimum, with its KKT certificate: stationarity relative to the problem's gradient scale (the interior point
    oracle's own termination measure: T = 25 with tight bounds reaches |c| ~ 1e3), primal feasibility absolute."""
    info = {}
    S, U, D, _ = oi.solve_ipm(prob, info=info)
    res, viol = onr.kkt_certificate(prob, S, U, D, act_tol=1e-6)
    assert res < 1e-7 * info["scale"] and viol < 1e-9, (res, info["scale"], viol)
    return S, U, D


@pytest.mark.parametrize("kin", KINS)
@pytest.mark.parametrize("T,M", SHAPES)
def test_oracle_solves_every_shape(T, M, kin):
    cfg = case_config(kin, T, M)
    _, _, probs = build_case(cfg, case_inputs(cfg, B=2))
    for prob in probs:
        _certified(prob)


@pytest.mark.parametrize("kin", KINS)
@pytest.mark.parametrize("regime", list(REGIMES))
def test_bound_regimes_have_their_active_families(regime, kin):
    """At every representative shape: the oracle's optimum is certified and the families the regime claims are active."""
    for T, M in REPRESENTATIVE:
        cfg = case_config(kin, T, M, regime)
        inp = case_inputs(cfg)
        _, _, probs = build_case(cfg, inp)
        total = dict.fromkeys(FAMILIES, 0)
        for prob in probs:
            S, U, D = _certified(prob)
            for k, v in active_counts(prob, U, D).items():
                total[k] += v
            if regime == "d_min_negative":
                assert D.min() >= -1e-12 and prob.d_min < 0
        missing = [f for f in REGIMES[regime] if total[f] == 0]
        assert not missing, (T, M, missing, total)


def test_dispatch_mirror_is_covered():
    """Every instantiation is reached by SHAPES, REPRESENTATIVE holds one shape of each, and the table sits on both sides of each
    switch: T = 16 | 17 and, among the generic T <= 16 instantiations, the largest TM of each HPL bucket and a TM of the next."""
    assert {instantiation(T, M) for T, M in SHAPES} == ALL_INSTANTIATIONS
    assert sorted(instantiation(T, M) for T, M in REPRESENTATIVE) == sorted(ALL_INSTANTIATIONS)
    tms = {T * M for T, M in SHAPES if T <= 16 and (T, M) not in ((10, 10), (15, 10))}
    for top in (32, 64, 128, 160):
        assert top in tms and any(top < tm <= top + 32 for tm in tms), top
    assert {1, 16, 17, 32} <= {T for T, _ in SHAPES} and {1, 32} <= {M for _, M in SHAPES}
    assert any(T > 16 and T * M == 128 for T, M in SHAPES) and any(T > 16 and T * M > 128 for T, M in SHAPES)
    assert all(T * M <= 256 and M <= 32 for T, M in SHAPES)
