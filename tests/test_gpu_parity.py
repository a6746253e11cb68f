"""Parity of the CUDA path (through the C ABI, via neupan_b200.PAN) against the CPU oracle.

Tolerance: north_star's 1e-4 relative (relative to the magnitude of each output tensor, floor 1).

Methodology (DESIGN.md "parity methodology"): one PAN iteration is compared at a time ("teacher
forcing": both sides start from the same nominal trajectory).  The K-fold composition of PAN
iterations is chaotic in cluttered scenes -- the oracle itself moves by 1e-1 after 10 iterations
when A_t is perturbed by one float32 ulp -- so an end-to-end K=10 comparison can only be
statistical; test_end_to_end_* does that and reports the fraction of environments within
tolerance.  The discrete top-M selection makes even a single iteration discontinuous: when the
M-th and (M+1)-th closest points are closer than `TIE` in distance the environment is excused.
"""
import numpy as np
import pytest
import torch

from gpu_helpers import make_pan, record, run_pan, to_cuda
from helpers import CONFIGS, GOLDEN, make_inputs, oracle_factory, rel_err, robot_spec, weights_path
from oracle import dune as od, ipm as oi, nrmp as onr

pytestmark = pytest.mark.gpu
TOL = 1e-4
TIE = 2e-5
# observed fractions of (env, iteration) pairs within TOL, minus 2 % (the rest are near-ties at the top-M boundary, each individually
# verified by _excused); `pytest -s` prints the observed fractions as OBSERVED lines
TEACHER_FORCED_MIN = {(c, s): 0.98 for c in ("C1", "C2", "C3", "C4", "C5") for s in ("annulus", "obstacles")}
E2E_K2_MIN = {"C2": 0.81, "C4": 0.98, "C5": 0.85}


def _oracle_dune(cfg, inp, b):
    rb, _ = robot_spec(cfg)
    w = od.load_weights(weights_path(cfg.model))
    G = torch.from_numpy(rb.G).float(); h = torch.from_numpy(rb.h).float()
    vel = None if inp["velocities"] is None else torch.from_numpy(inp["velocities"][b])
    p0, R, pl = od.point_flow(torch.from_numpy(inp["nom_s"][b]), torch.from_numpy(inp["points"][b]), vel, cfg.T, cfg.dt, 10 ** 9)
    return od.dune_forward(w, G, h, p0, R, pl), h


@pytest.mark.parametrize("cname", ["C1", "C2", "C3", "C4", "C5"])
@pytest.mark.parametrize("dune_kernel", [4, 2])
def test_dune_half_matches_oracle(cname, dune_kernel):
    """DUNE kernel alone (the screening pipeline and the exact kernel on every point): the M closest points per
    (env, step), their mu, lam, distance."""
    cfg = CONFIGS[cname]
    B = 6
    inp = make_inputs(cfg, B=B)
    pan = make_pan(cfg, K=1, max_envs=B, dune_kernel=dune_kernel)
    run_pan(pan, inp)
    sel = {k: v.cpu().numpy() for k, v in pan.read_selection().items()}
    # NOTE: selections are those of the (single) executed iteration, computed from the input nom_s
    worst = dict(mu=0.0, lam=0.0, dist=0.0)
    # mu / lam tolerance: north_star's 1e-4, relative to the largest entry of the (M, E) / (M, 2) block of the step
    MU_RTOL = 1e-4
    for b in range(B):
        (mu, lam, sp, md, dist), _ = _oracle_dune(cfg, inp, b)
        M = cfg.M
        for t in range(cfg.T + 1):
            d_sorted = np.sort(dist[t].numpy())
            assert np.allclose(sel["distance"][b, t], d_sorted[:M], rtol=1e-4, atol=2e-5)
            if d_sorted[M] - d_sorted[M - 1] < TIE or np.min(np.diff(d_sorted[:M + 1])) < TIE:
                continue  # near-tie: order / membership legitimately ambiguous at float32 accuracy
            assert np.allclose(sel["points"][b, t], sp[t][:, :M].T.numpy(), atol=1e-6)
            mu_o, lam_o = mu[t][:, :M].T.numpy(), lam[t][:, :M].T.numpy()
            worst["mu"] = max(worst["mu"], float(np.abs(sel["mu"][b, t] - mu_o).max() / max(1e-3, np.abs(mu_o).max())))
            worst["lam"] = max(worst["lam"], float(np.abs(sel["lam"][b, t] - lam_o).max() / max(1e-3, np.abs(lam_o).max())))
            worst["dist"] = max(worst["dist"], float(np.abs(sel["distance"][b, t] - d_sorted[:M]).max()))
        assert abs(pan.min_distance[b].item() - float(md)) < 2e-5
    record("dune_half", config=cname, dune_kernel=dune_kernel, mu_rel_to_row_max=worst["mu"], lam_rel_to_row_max=worst["lam"], dist_abs=worst["dist"])
    assert worst["mu"] < MU_RTOL and worst["lam"] < MU_RTOL, worst


@pytest.mark.parametrize("cname", ["C1", "C2", "C3", "C4", "C5"])
def test_nrmp_half_matches_oracle(cname):
    """NRMP kernel alone on explicit (fa, fb): the convex program's solution vs the float64 IPM oracle."""
    import ctypes as C

    from neupan_b200 import _lib

    cfg = CONFIGS[cname]
    B = 8
    inp = make_inputs(cfg, B=B, N=min(cfg.N, 120))
    rb, spec = robot_spec(cfg)
    fa = np.zeros((B, cfg.T, cfg.M, 2), np.float32); fb = np.zeros((B, cfg.T, cfg.M), np.float32)
    probs = []
    for b in range(B):
        (mu, lam, sp, md, dist), h = _oracle_dune(cfg, inp, b)
        a, c = od.nrmp_coefficients(h, mu, lam, sp, cfg.T, cfg.M)
        fa[b], fb[b] = a.numpy(), c.numpy()
        probs.append(onr.build_problem(spec, onr.Adjust(**cfg.adjust), inp["nom_s"][b], inp["nom_u"][b], inp["ref_s"][b], inp["ref_us"][b], fa[b], fb[b], cfg.M))
    pan = make_pan(cfg, K=1, max_envs=B)
    lib = pan._ensure_handle(B, cfg.N)
    t = to_cuda(dict(nom_s=inp["nom_s"], nom_u=inp["nom_u"], ref_s=inp["ref_s"], ref_us=inp["ref_us"], fa=fa, fb=fb))
    oS = torch.empty_like(t["nom_s"]); oU = torch.empty_like(t["nom_u"]); oD = torch.empty(B, cfg.T, device="cuda"); st = torch.empty(B, dtype=torch.int32, device="cuda")
    p = lambda x: C.c_void_p(x.data_ptr())
    _lib.check(lib.nb_nrmp_forward(pan._handle, B, p(t["nom_s"]), p(t["nom_u"]), p(t["ref_s"]), p(t["ref_us"]), p(t["fa"]), p(t["fb"]),
                                   p(oS), p(oU), p(oD), p(st), None))
    torch.cuda.synchronize()
    assert (st.cpu().numpy() == 0).all()
    for b in range(B):
        S, U, D, _ = oi.solve_ipm(probs[b])
        assert rel_err(oS[b].cpu().numpy(), S) < TOL and rel_err(oU[b].cpu().numpy(), U) < TOL and rel_err(oD[b].cpu().numpy(), D[0]) < TOL
        # tighter: the kernel runs the same FP64 method, so it should agree to float32 rounding
        assert np.abs(oU[b].cpu().numpy() - U).max() < 5e-6
        res, viol = onr.kkt_certificate(probs[b], oS[b].cpu().numpy().astype(np.float64), oU[b].cpu().numpy().astype(np.float64), oD[b].cpu().numpy().astype(np.float64), act_tol=1e-5)
        assert viol < 1e-5


def _excused(cfg, inp, b, s, u):
    """True if the single iteration from (s,u) has a near-tie at the selection boundary for env b."""
    one = {k: (None if v is None else v[b:b + 1]) for k, v in inp.items()}
    one = dict(one, nom_s=s[None], nom_u=u[None])
    (mu, lam, sp, md, dist), _ = _oracle_dune(cfg, one, 0)
    for t in range(cfg.T + 1):
        d = np.sort(dist[t].numpy())
        if d.shape[0] > cfg.M and d[cfg.M] - d[cfg.M - 1] < 5 * TIE:
            return True
    return False


@pytest.mark.parametrize("cname", ["C1", "C2", "C3", "C4", "C5"])
@pytest.mark.parametrize("scene", ["annulus", "obstacles"])
def test_single_iteration_teacher_forced_vs_golden(cname, scene):
    """Each PAN iteration, started from the committed oracle trace, reproduces the next trace entry."""
    cfg = CONFIGS[cname]
    z = np.load(f"{GOLDEN}/oracle_pan_{cname}_{scene}.npz")
    nenv, K = int(z["n_env"]), int(z["K"])
    inp = make_inputs(cfg, B=nenv, scene=scene)
    pan = make_pan(cfg, K=1, max_envs=nenv)
    s, u = inp["nom_s"], inp["nom_u"]
    checked, worst_ok = 0, 0.0
    for k in range(K):
        S, U, D, md = run_pan(pan, dict(inp, nom_s=s, nom_u=u))
        for b in range(nenv):
            err = max(rel_err(S[b], z["S"][b, k]), rel_err(U[b], z["U"][b, k]), rel_err(D[b], z["D"][b, k, 0]), abs(md[b] - z["min_distance"][b, k]))
            if err < TOL:
                checked += 1
                worst_ok = max(worst_ok, err)
            else:  # only a near-tie at the top-M boundary may excuse a mismatch
                assert _excused(cfg, inp, b, s[b], u[b]), (k, b, err)
        s, u = np.ascontiguousarray(z["S"][:, k]), np.ascontiguousarray(z["U"][:, k])
    frac = checked / (nenv * K)
    record("teacher_forced", config=cname, scene=scene, pairs=nenv * K, within_tol=checked, fraction=frac, worst_accepted_err=worst_ok)
    # ratchet: thresholds = observed minus 2 %
    assert frac >= TEACHER_FORCED_MIN[(cname, scene)], f"only {checked}/{nenv * K} (env, iteration) pairs within {TOL}"


@pytest.mark.parametrize("cname,B", [("C2", 24), ("C4", 24), ("C5", 8)])
def test_end_to_end_two_iterations_vs_live_oracle(cname, B):
    """iter_num = 2 (the reference's default, every example yaml): full forward vs the oracle.

    Statistical by necessity: one PAN iteration amplifies a perturbation of its nominal input by
    10-40x in some scenes (measured on the oracle itself, tests/test_oracle_nrmp.py::
    test_oracle_iteration_amplifies_perturbations), so the ~1e-5 float32-level difference after
    iteration 1 can exceed 1e-4 after iteration 2 although each iteration on its own matches to
    1e-4 (test_single_iteration_teacher_forced_vs_golden)."""
    cfg = CONFIGS[cname]
    inp = make_inputs(cfg, B=B, scene="obstacles")
    pan = make_pan(cfg, K=2, max_envs=B)
    S, U, D, md = run_pan(pan, inp)
    from oracle import pan as op
    So, Uo, Do, mdo, _ = op.run_batch(oracle_factory(cfg, K=2), inp)
    err = np.array([max(rel_err(S[b], So[b]), rel_err(U[b], Uo[b]), rel_err(D[b], Do[b, 0]), abs(md[b] - mdo[b])) for b in range(B)])
    record("e2e_k2", config=cname, envs=B, within_tol=int(np.sum(err < TOL)), fraction=float(np.mean(err < TOL)), within_50tol=float(np.mean(err < 50 * TOL)),
           max_err=float(err.max()), median_err=float(np.median(err)))
    assert np.mean(err < TOL) >= E2E_K2_MIN[cname], f"{np.sum(err < TOL)}/{B} environments within {TOL}"
    # a top-M membership flip in iteration 2 (near-tie at the M-th distance after the 1e-5 drift of iteration 1) moves a
    # single environment by 1e-2..1e-1; tools/diag_e2e.py shows both of its iterations match to 2e-5 when teacher-forced
    assert np.mean(err < 50 * TOL) >= 0.85
    assert (pan.iterations.cpu().numpy() == 2).all() and (pan.status.cpu().numpy() == 0).all()


def test_end_to_end_k10_vs_live_oracle_reported():
    """The benchmarked setting (C4, K = 10) end to end against the oracle.  Ten chaotic iterations (see the module docstring):
    what is asserted is the part that is stable -- min_distance of iteration-1 quantities, status, iteration count, feasibility --
    and the observed agreement fraction is recorded (not hidden) for DESIGN.md."""
    cfg = CONFIGS["C4"]
    B = 16
    inp = make_inputs(cfg, B=B, scene="obstacles")
    pan = make_pan(cfg, K=10, max_envs=B)
    S, U, D, md = run_pan(pan, inp)
    from oracle import pan as op
    So, Uo, Do, mdo, _ = op.run_batch(oracle_factory(cfg, K=10), inp)
    err = np.array([max(rel_err(S[b], So[b]), rel_err(U[b], Uo[b]), rel_err(D[b], Do[b, 0])) for b in range(B)])
    record("e2e_k10", config="C4", envs=B, within_tol=int(np.sum(err < TOL)), fraction=float(np.mean(err < TOL)), within_100tol=float(np.mean(err < 100 * TOL)),
           max_err=float(err.max()), median_err=float(np.median(err)))
    assert (pan.iterations.cpu().numpy() == 10).all() and (pan.status.cpu().numpy() == 0).all()
    assert np.median(err) < 100 * TOL


def test_c4_env_934_iteration_5():
    """The environment whose 5th NRMP instance broke round 1's CPU oracle (cost gradient O(1e3), absolute residual test):
    the GPU solve of exactly that instance, teacher-forced from the oracle's trace, must be status 0 and match."""
    cfg = CONFIGS["C4"]
    inp = make_inputs(cfg, B=1, env_offset=934)
    o = oracle_factory(cfg, K=5)()
    o.forward(inp["nom_s"][0], inp["nom_u"][0], inp["ref_s"][0], inp["ref_us"][0], inp["points"][0], inp["velocities"][0], keep_trace=True)
    assert o.fallbacks == 0 and len(o.trace) == 5
    pan = make_pan(cfg, K=1, max_envs=1)
    S, U, D, md = run_pan(pan, dict(inp, nom_s=o.trace[3]["S"][None], nom_u=o.trace[3]["U"][None]))
    assert int(pan.status.cpu()[0]) == 0
    err = max(rel_err(S[0], o.trace[4]["S"]), rel_err(U[0], o.trace[4]["U"]), rel_err(D[0], o.trace[4]["D"][0]))
    record("c4_env_934_it5", err=err, ipm_iterations=int(pan.ipm_iterations.cpu()[0]))
    assert err < TOL


@pytest.mark.parametrize("cname", ["C1", "C2", "C4", "C5"])
def test_single_iteration_vs_reference_pan_golden(cname):
    """Directly against the REFERENCE'S OWN PAN.forward (tests/golden/ref_pan.npz, made by make_golden_refpan.py: pan.py / dune.py /
    nrmp.py / robot.py executing unmodified, cvxpy + cvxpylayers replaced by the numeric shim): one PAN iteration per environment."""
    z = np.load(f"{GOLDEN}/ref_pan.npz")
    cfg = CONFIGS[cname]
    S0, N = z[f"{cname}_S"], int(z[f"{cname}_N"])
    nenv = S0.shape[0]
    inp = make_inputs(cfg, B=nenv, N=N, scene="obstacles")
    pan = make_pan(cfg, K=1, N=N, max_envs=nenv)
    S, U, D, md = run_pan(pan, inp)
    err = [max(rel_err(S[b], S0[b]), rel_err(U[b], z[f"{cname}_U"][b]), rel_err(D[b], z[f"{cname}_D"][b][0]), abs(md[b] - z[f"{cname}_md"][b])) for b in range(nenv)]
    record("vs_reference_pan_golden", config=cname, envs=nenv, max_err=float(max(err)))
    bad = [b for b in range(nenv) if err[b] >= TOL and not _excused(cfg, inp, b, inp["nom_s"][b], inp["nom_u"][b])]
    assert not bad, (bad, err)


def test_default_two_iterations_vs_reference_pan_golden():
    """BASELINE config 1 with the reference's default iter_num = 2: the whole forward against the reference's own PAN.forward
    (golden through the shim).  Two chained iterations: statistical like test_end_to_end_two_iterations_vs_live_oracle."""
    z = np.load(f"{GOLDEN}/ref_pan.npz")
    cfg = CONFIGS["C1"]
    inp = make_inputs(cfg, B=6, N=100, scene="obstacles")
    S, U, D, md = run_pan(make_pan(cfg, K=2, N=100, max_envs=6), inp)
    err = np.array([max(rel_err(S[b], z["C1k2_S"][b]), rel_err(U[b], z["C1k2_U"][b]), rel_err(D[b], z["C1k2_D"][b][0]), abs(md[b] - z["C1k2_md"][b])) for b in range(6)])
    record("vs_reference_pan_golden_k2", config="C1", envs=6, within_tol=int((err < TOL).sum()), max_err=float(err.max()))
    assert (err < TOL).mean() >= 0.8 and np.median(err) < TOL


def test_host_and_device_entry_points_agree():
    cfg = CONFIGS["C2"]
    inp = make_inputs(cfg, B=5)
    a = run_pan(make_pan(cfg, K=2, max_envs=5), inp, cuda=True)
    b = run_pan(make_pan(cfg, K=2, max_envs=5), inp, cuda=False)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_unbatched_call_matches_batched():
    cfg = CONFIGS["C1"]
    inp = make_inputs(cfg, B=1)
    pan = make_pan(cfg, max_envs=1)
    S, U, D, md = run_pan(pan, inp)
    pan2 = make_pan(cfg, max_envs=1)
    t = to_cuda(inp)
    s1, u1, d1 = pan2(t["nom_s"][0], t["nom_u"][0], t["ref_s"][0], t["ref_us"][0], t["points"][0], None)
    assert s1.shape == (3, cfg.T + 1) and u1.shape == (2, cfg.T) and d1.shape == (1, cfg.T)
    assert np.array_equal(s1.cpu().numpy(), S[0]) and np.array_equal(u1.cpu().numpy(), U[0])
    assert pan2.min_distance.dim() == 0 and pan2.dune_points.shape == (2, cfg.N) and pan2.nrmp_points.shape == (2, cfg.M)
