"""The float64 chain gradient (oracle/nrmp_grad.backward_chain) against central differences of the frozen chain
(oracle/nrmp_grad.chain_loss) in the regimes the native adjoint meets beyond T = 10, M = 10 (tests/test_gpu_grad.py compares
the two): horizons with 2T > 32 up to the largest T the ABI accepts, no-obstacle mode (no D), a chain of one solve (an
environment that stops after its first PAN iteration), clouds with fewer points than M or none, and omni with a vector q_s."""
import dataclasses

import numpy as np
import pytest

from helpers import CONFIGS, make_inputs, oracle_factory
from oracle import nrmp_grad as og


def _chain(cfg, env=0, K=2, N=80, n_points=None, adjust=None, M=None, iter_threshold=0.0, calls=1):
    """The NRMP problems of the LAST of ``calls`` OraclePAN.forward calls of one environment (one oracle, its stop-criterion
    state carried from call to call), with float64-consistent gamma_a / gamma_b.  ``n_points`` truncates the cloud (0: no points)."""
    inp = make_inputs(cfg, B=1, N=N, scene="obstacles", env_offset=env)
    pts, vel = inp["points"][0], None if inp["velocities"] is None else inp["velocities"][0]
    if n_points is not None:
        pts = pts[:, :n_points] if n_points else None
        vel = None if (vel is None or not n_points) else vel[:, :n_points]
    pan = oracle_factory(cfg, K=K, N=N, adjust=adjust, M=M, iter_threshold=iter_threshold)()
    orig = pan._solve
    for _ in range(calls):
        probs = []
        pan._solve = lambda prob, probs=probs: (probs.append(prob), orig(prob))[1]
        pan.forward(inp["nom_s"][0], inp["nom_u"][0], inp["ref_s"][0], inp["ref_us"][0], pts, vel)
    ref_s, ref_us = inp["ref_s"][0].astype(np.float64), inp["ref_us"][0].astype(np.float64)
    return [og.with_theta(p, ref_s, ref_us, og.theta_of(p)) for p in probs], ref_s, ref_us


def _weights(T, seed=2):
    rng = np.random.default_rng(seed)
    wS, wU, wD = rng.normal(size=(3, T + 1)), rng.normal(size=(2, T)), rng.normal(size=T)
    wS[:, 0] = 0.0  # the initial state is a constant
    return wS, wU, wD


def _check_against_fd(probs, ref_s, ref_us, min_checked=4):
    """backward_chain against central differences of chain_loss in each THETA component whose difference quotient is stable
    between two step sizes (the active-set-stability skip of tests/test_oracle_nrmp_grad.py: a kink inside the stencil).
    Returns (gradient, number of components checked)."""
    wS, wU, wD = _weights(probs[0].T)
    got = og.backward_chain(probs, ref_s, ref_us, wS, wU, wD)
    th0 = og.theta_of(probs[0])
    checked = 0
    for i in range(7):
        fd = []
        for rel in (1e-4, 1e-5):
            h = rel * max(1.0, abs(th0[i]))
            tp, tm = th0.copy(), th0.copy()
            tp[i] += h; tm[i] -= h
            fd.append((og.chain_loss(probs, ref_s, ref_us, tp, wS, wU, wD) - og.chain_loss(probs, ref_s, ref_us, tm, wS, wU, wD)) / (2 * h))
        if abs(fd[0] - fd[1]) > 1e-3 * max(1.0, abs(fd[0])):
            continue
        assert abs(got[i] - fd[1]) < 1e-3 * max(1.0, abs(fd[1])), (og.THETA[i], got[i], fd)
        checked += 1
    assert checked >= min_checked, checked
    assert np.abs(got).max() > 1e-3  # not a trivially zero gradient
    return got, checked


@pytest.mark.parametrize("T,M", [(17, 10), (32, 8)])
def test_long_horizons(T, M):
    """2T > 32: the adjoint keeps rows lane + 32 in a second register; T = 32 is the largest horizon of the ABI."""
    cfg = dataclasses.replace(CONFIGS["C4"], T=T, M=M, N=96)
    probs, ref_s, ref_us = _chain(cfg, env=0, K=2, N=96)
    assert len(probs) == 2 and probs[0].T == T and probs[0].M == M
    _check_against_fd(probs, ref_s, ref_us)


def test_no_obstacle_mode_has_no_distance_block():
    cfg = CONFIGS["C4"]
    probs, ref_s, ref_us = _chain(cfg, env=1, K=2, M=0)
    assert probs[0].M == 0
    got, _ = _check_against_fd(probs, ref_s, ref_us, min_checked=3)
    # eta, d_max and d_min act on D only: without D they have no gradient at all
    assert got[4] == 0.0 and got[5] == 0.0 and got[6] == 0.0


def test_chain_of_one_solve_from_an_early_stop():
    """The second forward of an oracle whose stop threshold is huge stops after its first iteration (the stored state of the first
    call is what it compares against): its chain has one solve, and the gradient is that solve's own."""
    cfg = CONFIGS["C5"]
    probs, ref_s, ref_us = _chain(cfg, env=2, K=4, iter_threshold=1e9, calls=2)
    assert len(probs) == 1
    got, _ = _check_against_fd(probs, ref_s, ref_us)
    wS, wU, wD = _weights(probs[0].T)
    single = og.backward(probs[0], ref_s, ref_us, wS, wU, wD)
    assert np.abs(got - single).max() <= 1e-12 * max(1.0, np.abs(single).max())


@pytest.mark.parametrize("n_points", [3, 0])
def test_sparse_clouds(n_points):
    """Fewer points than M (the remaining hinge rows are zero) and none at all (D without any hinge)."""
    cfg = CONFIGS["C4"]
    probs, ref_s, ref_us = _chain(cfg, env=3, K=2, N=80, n_points=n_points)
    assert probs[0].M == cfg.M
    if n_points == 0:
        assert not np.any(probs[0].fa) and not np.any(probs[0].fb)
    _check_against_fd(probs, ref_s, ref_us, min_checked=3)


def test_omni_vector_qs_has_no_heading_gradient():
    cfg = CONFIGS["C5"]
    adj = dict(cfg.adjust, q_s=[0.7, 1.3, 0.4])
    probs, ref_s, ref_us = _chain(cfg, env=1, K=2, adjust=adj)
    assert np.allclose(probs[0].q, [0.7, 1.3, 0.4])
    got, _ = _check_against_fd(probs, ref_s, ref_us)
    assert got[2] == 0.0  # the omni program has no heading term: q_s[2] does not enter it
    assert got[0] != 0.0 and got[1] != 0.0
