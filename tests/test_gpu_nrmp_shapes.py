"""The NRMP solve at every instantiation of nrmp_kernel that launch_nrmp (csrc/nrmp.cu) can pick, for the diff, acker and omni
robots, against the float64 interior point oracle; with tight, mixed-infinite and negative-d_min bounds, fewer points than M, no
obstacles at all, the status paths of the generic instantiations, and the persistent-warp schedule.  The case tables, the dispatch
mirror and the problem builder live in tests/test_oracle_nrmp_shapes.py, which checks them on the CPU.

nb_nrmp_forward runs on explicit (fa, fb) from the oracle's DUNE selection, so no near-tie excuses anything: every environment of
every case must pass the bars of test_gpu_parity.py::test_nrmp_half_matches_oracle (U[1]: U_ENERGY below).  Every launch whose
kernel name torch.profiler records must be the instantiation the mirror names, and each case must have one such record.
`pytest -s` prints the worst errors per instantiation and kinematics, the active row counts and the kernel names as OBSERVED
lines."""
import ctypes as C
import os
import re
from math import inf

import numpy as np
import pytest
import torch

from gpu_helpers import make_pan, record, run_pan, to_cuda
from helpers import make_inputs, rel_err
from oracle import ipm as oi, nrmp as onr
from test_gpu_grad import COMPONENT_TOL, MIN_COMPARED_SMALL, _check, _loss_backward, _oracle_env, _weights
from test_gpu_parity import TOL
from test_oracle_nrmp_shapes import (ALL_INSTANTIATIONS, FAMILIES, KINS, REGIMES, REPRESENTATIVE, SHAPES, active_counts, build_case,
                                     case_config, case_inputs, instantiation, label)

pytestmark = pytest.mark.gpu
U_ABS = 5e-6     # max |U[0] - U_oracle[0]| (the kernel runs the same FP64 method: float32 rounding)
VIOL = 1e-5      # primal violation of the KKT certificate at the kernel's (S, U, D)
# The second control (angular speed, steering angle, heading command) is weighted only through the heading or the positions it
# moves.  Without an active angular box its late horizon steps are a flat direction of the cost: the smallest eigenvalue of the cost
# Hessian in U is 4e-4 for the acker robot (q_s = 0.5, bk = 0.1, wheelbase 3 m).  Along it the cost is flat to 1e-9 of its value,
# and the kernel's termination test (dual residual < 1e-8 of the gradient scale) leaves U[1] up to 3e-4 from the optimum (acker),
# 1.2e-5 (diff and omni with an infinite angular box), on an H100; U[0] stays within 3e-7.  The bar of U[1] is therefore set in
# the norm the residual controls, sqrt(dU' P dU) with P the cost Hessian in U: observed <= 9e-6 (acker), <= 1.4e-6 elsewhere.
U_ENERGY = 2e-5
# The oracle is solved to a mean complementarity of 1e-13 instead of its default 1e-11: at 1e-11 it stops up to 1e-4 away from
# the optimum along the same flat directions (acker and omni with M = 0), which the kernel reaches.
ORACLE_TOL = 1e-13
GENERIC = [s for s in REPRESENTATIVE if instantiation(*s)[2] == 0]
_KERNEL = re.compile(r"nrmp_kernel<\s*(\d+),\s*(true|false),\s*(\d+),\s*(\d+)\s*>|nrmp_kernelILi(\d+)ELb([01])ELi(\d+)ELi(\d+)E")


def _kernels(prof):
    """(HPL, SMALL, TT, MM) of every nrmp_kernel launch torch.profiler recorded (demangled or mangled names)."""
    found = []
    for e in prof.events():
        m = _KERNEL.search(e.name)
        if m:
            g = m.groups()
            g = g[:4] if g[0] is not None else g[4:]
            found.append((int(g[0]), g[1] in ("true", "1"), int(g[2]), int(g[3])))
    return found


def _solve(cfg, inp, fa, fb, profile=False, pan=None):
    """nb_nrmp_forward on explicit coefficients (NULL when fa is None) for every environment of `inp`: dict of S, U, D, status,
    interior point iterations (numpy) and, with `profile`, the instantiations the profiler saw launched."""
    from neupan_b200 import _lib

    B = inp["nom_s"].shape[0]
    own = pan is None
    if own:
        pan = make_pan(cfg, K=1, max_envs=B, N=max(cfg.N, 1), dune_kernel=2)
    lib = pan._ensure_handle(B, 0)
    arrs = dict(nom_s=inp["nom_s"], nom_u=inp["nom_u"], ref_s=inp["ref_s"], ref_us=inp["ref_us"])
    if fa is not None:
        arrs.update(fa=fa, fb=fb)
    t = to_cuda(arrs)
    oS = torch.empty_like(t["nom_s"]); oU = torch.empty_like(t["nom_u"]); oD = torch.empty(B, cfg.T, device="cuda")
    st = torch.empty(B, dtype=torch.int32, device="cuda"); it = torch.empty(B, dtype=torch.int32, device="cuda")
    p = lambda x: C.c_void_p(x.data_ptr())
    pa = lambda k: p(t[k]) if k in t else None
    launch = lambda: _lib.check(lib.nb_nrmp_forward(pan._handle, B, p(t["nom_s"]), p(t["nom_u"]), p(t["ref_s"]), p(t["ref_us"]), pa("fa"),
                                                    pa("fb"), p(oS), p(oU), p(oD), p(st), None))
    kernels = None
    if profile:
        from torch.profiler import ProfilerActivity, profile as profiled

        # the profiler misses a launch now and then (a few of ~250 sessions on an H100, sometimes three in a row): the solve has no
        # state, so it is launched again under a new session, up to three times; the callers require one confirmation per case
        for _ in range(3):
            with profiled(activities=[ProfilerActivity.CUDA]) as prof:
                launch()
                torch.cuda.synchronize()
            kernels = _kernels(prof)
            if kernels:
                break
    else:
        launch()
    _lib.check(lib.nb_pan_read_diagnostics(pan._handle, B, p(it), None))
    torch.cuda.synchronize()
    out = dict(S=oS.cpu().numpy(), U=oU.cpu().numpy(), D=oD.cpu().numpy(), status=st.cpu().numpy(), iters=it.cpu().numpy(), kernels=kernels)
    if own:
        pan.close()
    return out


def _compare(probs, out):
    """Every environment against the oracle with the bars of test_nrmp_half_matches_oracle (U[1]: U_ENERGY); returns the worst
    errors and the active row counts at the oracle's optimum."""
    assert (out["status"] == 0).all(), out["status"]
    worst = dict(rel_err_s=0.0, rel_err_u=0.0, rel_err_d=0.0, max_abs_u0_err=0.0, max_abs_u1_err=0.0, u_err_cost_norm=0.0, max_kkt_violation=0.0)
    active = dict.fromkeys(FAMILIES, 0)
    for b, prob in enumerate(probs):
        S, U, D, _ = oi.solve_ipm(prob, tol=ORACLE_TOL, max_iter=120)
        gS, gU, gD = out["S"][b], out["U"][b], out["D"][b]
        dU = gU.astype(np.float64) - U
        P = oi.assemble(prob)["P"][:2 * prob.T, :2 * prob.T]
        x = dU.T.reshape(-1)  # time-major, the order of P
        e = dict(rel_err_s=rel_err(gS, S), rel_err_u=rel_err(gU, U), max_abs_u0_err=float(np.abs(dU[0]).max()),
                 max_abs_u1_err=float(np.abs(dU[1]).max()), u_err_cost_norm=float(np.sqrt(max(x @ P @ x, 0.0))))
        if D is None:
            assert (gD == 0).all(), b  # no obstacle rows: the kernel writes D = 0
        else:
            e["rel_err_d"] = rel_err(gD, D[0])
        _, viol = onr.kkt_certificate(prob, gS.astype(np.float64), gU.astype(np.float64), None if D is None else gD.astype(np.float64), act_tol=1e-5)
        e["max_kkt_violation"] = viol
        assert max(e["rel_err_s"], e["rel_err_u"], e.get("rel_err_d", 0.0)) < TOL and e["max_abs_u0_err"] < U_ABS, (b, e)
        assert e["u_err_cost_norm"] < U_ENERGY and viol < VIOL, (b, e)
        for k, v in e.items():
            worst[k] = max(worst[k], v)
        for k, v in active_counts(prob, U, D).items():
            active[k] += v
    return worst, active


def _run_case(kin, T, M, regime=None, **kw):
    cfg = case_config(kin, T, M, regime, **kw)
    inp = case_inputs(cfg)
    fa, fb, probs = build_case(cfg, inp)
    out = _solve(cfg, inp, fa, fb, profile=True)
    inst = instantiation(T, M)
    assert out["kernels"] in ([], [inst]), (T, M, out["kernels"], inst)
    worst, active = _compare(probs, out)
    return cfg, inp, fa, fb, out, worst, active


@pytest.mark.parametrize("T,M", SHAPES)
def test_every_instantiation_matches_the_oracle(T, M):
    """Each (T, M) of the table with the diff, acker and omni robot: six environments, every one within the bars."""
    confirmed = 0
    for kin in KINS:
        _, _, _, _, out, worst, active = _run_case(kin, T, M)
        confirmed += bool(out["kernels"])
        record("nrmp_shapes", kernel=label(instantiation(T, M)), kin=kin, T=T, M=M, envs=len(out["status"]),
               ipm_iterations_max=int(out["iters"].max()), **worst, active=active, profiled_kernel=[label(k) for k in out["kernels"]])
    assert confirmed, "the profiler saw none of the three launches"


@pytest.mark.parametrize("regime", list(REGIMES))
@pytest.mark.parametrize("T,M", REPRESENTATIVE)
def test_bound_regimes_match_the_oracle(T, M, regime):
    """One shape per instantiation under each bound regime: tight bounds (every constraint family active somewhere), one of speed /
    rate infinite on each control component, d_min < 0, and clouds of fewer points than M."""
    confirmed = 0
    for kin in KINS:
        cfg, inp, fa, fb, out, worst, active = _run_case(kin, T, M, regime)
        confirmed += bool(out["kernels"])
        record("nrmp_bound_regime", regime=regime, kernel=label(instantiation(T, M)), kin=kin, T=T, M=M, **worst, active=active,
               speed_bound=[float(v) for v in cfg.make_robot().max_speed.reshape(-1)], acce_bound=[float(v) for v in cfg.make_robot().max_acce.reshape(-1)])
        missing = [f for f in REGIMES[regime] if active[f] == 0]
        assert not missing, (kin, missing, active)
        if regime == "d_min_negative":
            # the program uses max(d_min, 0): the same bits as d_min = 0
            ref = _solve(case_config(kin, T, M, adjust=dict(d_min=0.0)), inp, fa, fb)
            for k in ("S", "U", "D", "status", "iters"):
                assert np.array_equal(out[k], ref[k]), k
    assert confirmed, "the profiler saw none of the three launches"


@pytest.mark.parametrize("kin", KINS)
@pytest.mark.parametrize("T", [1, 8, 16, 17, 32])
def test_no_obstacles(T, kin):
    """M = 0 (no obstacle rows, null coefficients): <1, true> at T <= 16 runs without the DMMA assembly, on the pair-table path;
    <4, false> at T > 16."""
    cfg, inp, fa, fb, out, worst, active = _run_case(kin, T, 0, N=0)
    assert fa is None
    record("nrmp_no_obstacles", kernel=label(instantiation(T, 0)), kin=kin, T=T, **worst, ipm_iterations_max=int(out["iters"].max()))


@pytest.mark.parametrize("T,M", GENERIC)
def test_singular_last_pivot_is_reported(T, M):
    """The diff robot with nothing that weighs its last angular velocity (q_s[2] = 0, bk = 0, no angular speed or acceleration bound):
    the last row of the reduced Hessian is exactly zero.  SMALL factors two columns per step and exits at the second; the other
    factorisation exits at its one column.  Either way: NB_STATUS_NUMERIC and the nominal trajectory back bit for bit."""
    cfg = case_config("diff", T, M, robot=dict(max_speed=[8, inf], max_acce=[8, inf]), adjust=dict(q_s=[1.0, 1.0, 0.0], bk=0.0))
    inp = case_inputs(cfg)
    fa, fb, _ = build_case(cfg, inp)
    out = _solve(cfg, inp, fa, fb)
    assert (out["status"] == 2).all(), out["status"]
    assert np.array_equal(out["S"], inp["nom_s"]) and np.array_equal(out["U"], inp["nom_u"])


def test_infeasible_distance_bounds_are_reported():
    """d_min > d_max at a generic shape: NB_STATUS_INFEASIBLE, no iteration, the nominal trajectory back."""
    for kin in KINS:
        cfg = case_config(kin, 20, 6, adjust=dict(d_max=0.2, d_min=0.5))
        inp = case_inputs(cfg)
        fa, fb, _ = build_case(cfg, inp)
        out = _solve(cfg, inp, fa, fb)
        assert (out["status"] == 4).all() and (out["iters"] == 0).all(), (kin, out["status"])
        assert np.array_equal(out["S"], inp["nom_s"]) and np.array_equal(out["U"], inp["nom_u"])


@pytest.mark.parametrize("T,M", GENERIC)
def test_persistent_schedule_is_bitwise_invariant(T, M):
    """8 distinct problems, replicated in a shuffled order into B = 64 x SMs + 64 environments.  A generic instantiation runs at most
    2 warps per CTA and an SM holds at most 32 CTAs, so at most 64 x SMs warps are resident: the batch exceeds them and the launcher
    takes the persistent-warp schedule (CTAs pull environments from a counter).  Every copy equals the 8-environment run bit for bit
    (S, U, D, status, interior point iterations); so does the static environment -> warp map (NB_NRMP_STATIC=1, read when the handle
    is created)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = 64 * sms + 64
    kin = KINS[(T + M) % 3]
    cfg = case_config(kin, T, M, "tight")
    inp = case_inputs(cfg, B=8)
    fa, fb, _ = build_case(cfg, inp)
    idx = np.random.default_rng(T * 100 + M).permutation(np.arange(B) % 8)
    big = {k: None if v is None else np.ascontiguousarray(v[idx]) for k, v in inp.items()}
    small = _solve(cfg, inp, fa, fb)
    assert (small["status"] == 0).all()
    for static in (False, True):
        if static:
            os.environ["NB_NRMP_STATIC"] = "1"
        try:
            out = _solve(cfg, big, fa[idx], fb[idx])
        finally:
            os.environ.pop("NB_NRMP_STATIC", None)
        for k in ("S", "U", "D", "status", "iters"):
            assert np.array_equal(out[k], small[k][idx]), (static, k)
    record("nrmp_schedule", kernel=label(instantiation(T, M)), kin=kin, T=T, M=M, envs=B, distinct=8,
           ipm_iterations=[int(v) for v in small["iters"]])


# (T, M, kinematics) combinations no other test runs through PAN
PAN_CASES = [(8, 8, "acker"), (16, 16, "omni"), (20, 6, "acker"), (10, 10, "omni"), (15, 10, "diff"), (15, 10, "acker")]


@pytest.mark.parametrize("T,M,kin", PAN_CASES)
def test_pan_warm_start_reaches_the_cold_start_optimum(T, M, kin):
    """NB_OPT_NRMP_WARM through PAN: the warm record's layout depends on T, M and HPL.  Bar of
    test_gpu_features.py::test_nrmp_warm_start_reaches_the_cold_start_optimum."""
    cfg = case_config(kin, T, M)
    B = 32
    inp = case_inputs(cfg, B=B)
    pw, pc = make_pan(cfg, K=2, max_envs=B, nrmp_warm=1), make_pan(cfg, K=2, max_envs=B, nrmp_warm=0)
    a, b = run_pan(pw, inp), run_pan(pc, inp)
    iw, ic = pw.ipm_iterations.cpu().numpy(), pc.ipm_iterations.cpu().numpy()
    err = max(float(np.abs(a[i] - b[i]).max()) for i in range(3))
    record("nrmp_shapes_warm_vs_cold", kernel=label(instantiation(T, M)), kin=kin, T=T, M=M, max_abs_diff=err,
           ipm_iterations_warm=float(iw.mean()), ipm_iterations_cold=float(ic.mean()))
    assert (pw.status.cpu().numpy() == 0).all() and (pc.status.cpu().numpy() == 0).all()
    assert err < 5e-5, err


@pytest.mark.parametrize("T,M,kin", PAN_CASES)
def test_pan_gradients_match_the_oracle_chain(T, M, kin):
    """Differentiable mode through PAN (the forward kernel writes the adjoint record) against the float64 chain, with the rule of
    test_gpu_grad.py::_check.  Clouds of exactly M points: every point is selected at every step, so no top-M near-tie can send the
    GPU and the oracle down different chains (with 96 points, the acker cases had forwards comparable in only 3 and 4 of 6
    environments)."""
    B, K, N = 12, 2, M
    cfg = case_config(kin, T, M, N=N)
    inp = make_inputs(cfg, B=B, N=N, scene="obstacles")
    pan = make_pan(cfg, K=K, N=N, max_envs=B)
    w = _weights(T, B)
    t = to_cuda(inp)
    with torch.enable_grad():  # recording autograd is what puts PAN.forward in differentiable mode
        out = pan(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"])
        got = _loss_backward(pan, *out, w)
    assert (pan.status.cpu().numpy() == 0).all()
    oracles = [_oracle_env(cfg, inp, b, K, N) for b in range(B)]
    # the squared hinge (rho/2) max(0, r)^2 has no second derivative at r = 0, so the solution's derivative jumps there: a chain with
    # a hinge argument within KINK of zero has two valid gradients (diff at (15, 10), environment 3: |r| = 1.1e-4, gradients 25 %
    # apart).  Such environments are left out; of the others, MIN_COMPARED_SMALL must be compared, and at least half of the batch.
    KINK = 1e-3
    envs = [b for b in range(B) if _hinge_margin(oracles[b]["probs"]) >= KINK]
    # acker: the gradients pass through the flat steering direction of U_ENERGY's comment; per component 6.2e-3 observed at (15, 10)
    # (environment rule 3.7e-4), the per-component tolerance of the large-batch obstacle sweep of test_gpu_grad.py is the precedent
    comp_tol = 1e-2 if kin == "acker" else COMPONENT_TOL
    compared = _check("nrmp_shapes_backward", pan, out, got, w, envs, [oracles[b] for b in envs], 0.0, comp_tol=comp_tol,
                      kernel=label(instantiation(T, M)), kin=kin, T=T, M=M, at_hinge_kink=B - len(envs))
    assert len(compared) >= MIN_COMPARED_SMALL * len(envs) and 2 * len(compared) >= B, compared


def _hinge_margin(probs):
    """Smallest |hinge argument| at the oracle's optimum over the NRMP problems of one chain."""
    margin = np.inf
    for prob in probs:
        S, U, D, _ = oi.solve_ipm(prob)
        a = oi.assemble(prob)
        margin = min(margin, float(np.abs(a["J"] @ np.concatenate([U.T.reshape(-1), D.reshape(-1)]) + a["k"]).min()))
    return margin


def test_every_instantiation_and_kinematics_is_in_the_tables():
    """The tables above reach all nine instantiations with every kinematics."""
    assert {instantiation(T, M) for T, M in SHAPES} == ALL_INSTANTIATIONS
    assert {instantiation(T, 0) for T in (1, 8, 16, 17, 32)} == {(1, True, 0, 0), (4, False, 0, 0)}
