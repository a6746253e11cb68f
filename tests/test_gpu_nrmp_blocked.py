"""The NRMP solve of the compile-time specialisations (C4: T = 10, C5: T = 15) factors the reduced Newton system blocked, in the
DMMA accumulators that assemble it (nrmp_kernel.cuh, nrmp_block_cholesky).  Checks at full cloud size against the float64 oracle,
the `bad` path of a pivot in the identity-padded last block of C4, and the gradients of differentiable mode."""
import dataclasses
from math import inf

import numpy as np
import pytest
import torch

from gpu_helpers import make_pan, record, run_pan, to_cuda
from helpers import CONFIGS, make_inputs, rel_err, robot_spec
from oracle import dune as od, ipm as oi, nrmp as onr
from test_gpu_grad import MIN_COMPARED_SMALL, _check, _loss_backward, _oracle_env, _weights
from test_gpu_parity import TOL, _oracle_dune

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cname,offset", [("C4", 0), ("C4", 1000), ("C5", 0), ("C5", 700)])
def test_blocked_nrmp_matches_oracle_at_full_cloud(cname, offset):
    """nb_nrmp_forward on explicit (fa, fb) from the oracle's selection of the full cloud, against the float64 interior point
    oracle, with the bars of test_gpu_parity.py::test_nrmp_half_matches_oracle."""
    import ctypes as C

    from neupan_b200 import _lib

    cfg = CONFIGS[cname]
    B = 6
    inp = make_inputs(cfg, B=B, env_offset=offset)
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
    worst_u, worst_viol = 0.0, 0.0
    for b in range(B):
        S, U, D, _ = oi.solve_ipm(probs[b])
        assert rel_err(oS[b].cpu().numpy(), S) < TOL and rel_err(oU[b].cpu().numpy(), U) < TOL and rel_err(oD[b].cpu().numpy(), D[0]) < TOL
        du = float(np.abs(oU[b].cpu().numpy() - U).max())
        res, viol = onr.kkt_certificate(probs[b], oS[b].cpu().numpy().astype(np.float64), oU[b].cpu().numpy().astype(np.float64),
                                        oD[b].cpu().numpy().astype(np.float64), act_tol=1e-5)
        worst_u, worst_viol = max(worst_u, du), max(worst_viol, viol)
        assert du < 5e-6 and viol < 1e-5, (b, du, viol)
    record("nrmp_blocked_vs_oracle", config=cname, env_offset=offset, envs=B, max_abs_u_err=worst_u, max_kkt_violation=worst_viol)


def test_singular_pivot_in_padded_last_block_is_reported():
    """C4 (2T = 20: block rows 16..19 plus four identity rows) with nothing that weighs the last angular velocity: no cost on the
    heading (q_s[2] = 0, bk = 0) and no bound on the angular speed or acceleration.  Row 19 of the reduced Hessian is then exactly
    zero, its pivot is 0, and the solve must give up with NB_STATUS_NUMERIC and hand back the nominal trajectory."""
    cfg = CONFIGS["C4"]
    cfg = dataclasses.replace(cfg, robot_kwargs=dict(cfg.robot_kwargs, max_speed=[8, inf], max_acce=[8, inf]),
                              adjust=dict(cfg.adjust, q_s=[1.0, 1.0, 0.0], bk=0.0))
    B, N = 4, 120
    inp = make_inputs(cfg, B=B, N=N)
    pan = make_pan(cfg, K=1, N=N, max_envs=B)
    S, U, D, _ = run_pan(pan, inp)
    assert (pan.status.cpu().numpy() == 2).all()
    assert np.array_equal(S, inp["nom_s"]) and np.array_equal(U, inp["nom_u"])


@pytest.mark.parametrize("cname", ["C4", "C5"])
def test_blocked_nrmp_gradients_at_full_cloud(cname):
    """Differentiable mode: the factor saved for the adjoint (the `finishing` active-set system) comes from the blocked
    factorisation; nb_pan_backward against the float64 chain with the bounds of test_gpu_grad.py, at the full cloud size."""
    cfg = CONFIGS[cname]
    B, K = 4, 2
    inp = make_inputs(cfg, B=B, scene="obstacles")
    pan = make_pan(cfg, K=K, max_envs=B)
    t = to_cuda(inp)
    w = _weights(cfg.T, B, seed=11)
    with torch.enable_grad():  # recording autograd is what puts PAN.forward in differentiable mode
        out = pan(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"])
        per_env = _loss_backward(pan, *out, w)
    oracles = [_oracle_env(cfg, inp, b, K, cfg.N) for b in range(B)]
    _check("nrmp_blocked_backward", pan, out, per_env, w, range(B), oracles, MIN_COMPARED_SMALL, config=cname, K=K)
    assert np.abs(per_env).max() > 1e-3
