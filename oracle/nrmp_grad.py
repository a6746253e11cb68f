"""Sensitivity of the NRMP solution to the adjust parameters (TEST INFRASTRUCTURE; groundwork for SURVEY 8f row 3).

LON (example/LON/LON_corridor.py:21-35, 94-95, 121-127) back-propagates a loss on ``info["distance_tensor"]`` etc. through
``CvxpyLayer`` (nrmp.py:144) into the leaf parameters ``q_s, p_u, eta, d_max, d_min`` (nrmp.py:79-104).  This file is the
float64 statement of what that backward pass computes -- d(S, U, D)/d(theta) by implicit differentiation of the optimality
conditions of the condensed program (oracle/ipm.py: ``assemble``) at the solution, under strict complementarity:

    H dx + A_act' dlam = -(dP/dtheta x + dc/dtheta),   A_act dx = db_act/dtheta,   H = P + rho J_act' J_act

with A_act the active rows of ``Ab x <= bb`` and J_act the hinge rows with positive argument.  ``gamma_a = q_s * ref_s`` and
``gamma_b = p_u * ref_us`` (nrmp.py:156-159) are functions of the leaves, so their dependence is part of dc/dtheta.  It is
validated against central finite differences of the float64 interior point solver (tests/test_oracle_nrmp_grad.py).  No product
code exists for this row yet; nothing outside tests/ may import this module.
"""
from __future__ import annotations

import dataclasses

import numpy as np

from . import ipm
from .nrmp import NrmpProblem

THETA = ("q_s[0]", "q_s[1]", "q_s[2]", "p_u", "eta", "d_max", "d_min")


def theta_of(p: NrmpProblem) -> np.ndarray:
    return np.array([p.q[0], p.q[1], p.q[2], p.p_u, p.eta, p.d_max, p.d_min], dtype=np.float64)


def with_theta(p: NrmpProblem, ref_s: np.ndarray, ref_us: np.ndarray, theta: np.ndarray) -> NrmpProblem:
    """The same program with other adjust values, in float64 throughout (no float32 rounding of the parameter products:
    this is the smooth map whose derivative is wanted)."""
    q = np.asarray(theta[0:3], np.float64)
    return dataclasses.replace(p, q=q.copy(), p_u=float(theta[3]), eta=float(theta[4]), d_max=float(theta[5]), d_min=float(theta[6]),
                               gamma_a=q.reshape(3, 1) * np.asarray(ref_s, np.float64), gamma_b=float(theta[3]) * np.asarray(ref_us, np.float64).reshape(-1))


def _solve(p: NrmpProblem):
    """solve_ipm plus the solver's final multipliers and slacks (for active_sets)."""
    info = {}
    S, U, D, _ = ipm.solve_ipm(p, info=info)
    return S, U, D, info


def _x_of(p: NrmpProblem, U, D):
    x = np.asarray(U, np.float64).T.reshape(-1)  # time-major (u_{0,0}, u_{1,0}, u_{0,1}, ...)
    return np.concatenate([x, np.asarray(D, np.float64).reshape(-1)]) if p.M > 0 else x


def active_sets(p: NrmpProblem, x, tol=1e-7, info=None):
    """Active rows of Ab x <= bb and hinge rows with positive argument at x.  With the solver's ``info`` (solve_ipm), a row whose
    multiplier exceeds its slack is active too: a row held by a small multiplier ends the interior point iteration with a slack
    of gap / z (C4 without obstacles: 2e-7 at z ~ 5e-5), above any fixed slack tolerance."""
    m = ipm.assemble(p)
    slack = m["bb"] - m["Ab"] @ x
    act = slack < tol * (1.0 + np.abs(m["bb"]))
    if info is not None:
        act |= info["z_b"] > info["s_b"]
    hinge = (m["J"] @ x + m["k"]) > tol if p.M > 0 else np.zeros(0, bool)
    return act, hinge


def solution_sensitivity(p: NrmpProblem, ref_s, ref_us, tol=1e-7):
    """Returns dict(dS (7,3,T+1), dU (7,2,T), dD (7,T), active, hinge): derivatives of the optimal S, U, D w.r.t. THETA."""
    S, U, D, info = _solve(p)
    x = _x_of(p, U, D)
    m = ipm.assemble(p)
    act, hinge = active_sets(p, x, tol, info)
    A = m["Ab"][act]
    H = m["P"] + (m["rho"] * m["J"][hinge].T @ m["J"][hinge] if p.M > 0 else 0.0)
    n, na = m["n"], A.shape[0]
    K = np.zeros((n + na, n + na))
    K[:n, :n], K[:n, n:], K[n:, :n] = H, A.T, A
    th0 = theta_of(p)
    T, nU = p.T, m["nU"]
    dS, dU, dD = np.zeros((7, 3, T + 1)), np.zeros((7, 2, T)), np.zeros((7, T))
    for i in range(7):
        h = 1e-3 * max(1.0, abs(th0[i]))
        tp, tm = th0.copy(), th0.copy()
        tp[i] += h
        tm[i] -= h
        mp, mm = ipm.assemble(with_theta(p, ref_s, ref_us, tp)), ipm.assemble(with_theta(p, ref_s, ref_us, tm))
        # P is quadratic and c, bb are (bi)linear in theta: the central difference of these maps is exact up to rounding
        dg = ((mp["P"] @ x + mp["c"]) - (mm["P"] @ x + mm["c"])) / (2 * h)
        db = (mp["bb"] - mm["bb"])[act] / (2 * h)
        sol = np.linalg.lstsq(K, np.concatenate([-dg, db]), rcond=None)[0]
        dx = sol[:n]
        dU[i] = dx[:nU].reshape(T, 2).T
        if p.M > 0:
            dD[i] = dx[nU:]
        for t in range(T):
            dS[i, :, t + 1] = m["F"][t] @ dx[:nU]
    return dict(dS=dS, dU=dU, dD=dD, active=act, hinge=hinge, S=S, U=U, D=D)


def finite_difference(p: NrmpProblem, ref_s, ref_us, i: int, rel_step=1e-5):
    """Central difference of the float64 solve in THETA[i]; also reports whether the active sets agree on both sides."""
    th0 = theta_of(p)
    h = rel_step * max(1.0, abs(th0[i]))
    out, sets = [], []
    for sgn in (+1, -1):
        th = th0.copy()
        th[i] += sgn * h
        q = with_theta(p, ref_s, ref_us, th)
        S, U, D, info = _solve(q)
        out.append((S, U, D[0] if p.M > 0 else np.zeros(p.T)))
        sets.append(active_sets(q, _x_of(q, U, D), info=info))
    same = np.array_equal(sets[0][0], sets[1][0]) and np.array_equal(sets[0][1], sets[1][1])
    return tuple((a - b) / (2 * h) for a, b in zip(out[0], out[1])), same


def backward(p: NrmpProblem, ref_s, ref_us, gS, gU, gD, tol=1e-7):
    """Adjoint form (what a backward kernel would do: ONE linear solve per environment instead of one per parameter):
    given the upstream gradients dL/dS (3,T+1), dL/dU (2,T), dL/dD (T) returns dL/dtheta (7).
        g_x = F' dL/dS + dL/dU (+ dL/dD);   K' z = [g_x; 0];   dL/dtheta_i = z' [-(dP_i x + dc_i); db_act_i]"""
    S, U, D, info = _solve(p)
    x = _x_of(p, U, D)
    m = ipm.assemble(p)
    act, hinge = active_sets(p, x, tol, info)
    A = m["Ab"][act]
    H = m["P"] + (m["rho"] * m["J"][hinge].T @ m["J"][hinge] if p.M > 0 else 0.0)
    n, na, nU, T = m["n"], A.shape[0], m["nU"], p.T
    K = np.zeros((n + na, n + na))
    K[:n, :n], K[:n, n:], K[n:, :n] = H, A.T, A
    gx = np.zeros(n)
    gx[:nU] = np.asarray(gU, np.float64).T.reshape(-1)
    for t in range(T):
        gx[:nU] += m["F"][t].T @ np.asarray(gS, np.float64)[:, t + 1]
    if p.M > 0:
        gx[nU:] = np.asarray(gD, np.float64).reshape(-1)
    z = np.linalg.lstsq(K.T, np.concatenate([gx, np.zeros(na)]), rcond=None)[0]
    th0, out = theta_of(p), np.zeros(7)
    for i in range(7):
        h = 1e-3 * max(1.0, abs(th0[i]))
        tp, tm = th0.copy(), th0.copy()
        tp[i] += h
        tm[i] -= h
        mp, mm = ipm.assemble(with_theta(p, ref_s, ref_us, tp)), ipm.assemble(with_theta(p, ref_s, ref_us, tm))
        dg = ((mp["P"] @ x + mp["c"]) - (mm["P"] @ x + mm["c"])) / (2 * h)
        db = (mp["bb"] - mm["bb"])[act] / (2 * h)
        out[i] = z @ np.concatenate([-dg, db])
    return out


def backward_full(p: NrmpProblem, ref_s, ref_us, gS, gU, gD, tol=1e-7):
    """``backward`` plus the gradient that flows on into the previous PAN iteration: returns (dL/dtheta (7), dL/dpara_s (3,T+1)).
    ``para_s`` is the NRMP parameter the reference feeds with ``nom_s`` (nrmp.py:156, robot.py:243): the output S of the previous
    solve, a tensor that carries its autograd history.  It enters the program through the proximal term only
    (0.5 bk |S - para_s|^2, nrmp.py:350); its first column also pins S[:, 0], but that column is the same constant in every
    iteration, so its gradient is not needed (returned as zero)."""
    S, U, D, info = _solve(p)
    x = _x_of(p, U, D)
    m = ipm.assemble(p)
    act, hinge = active_sets(p, x, tol, info)
    A = m["Ab"][act]
    H = m["P"] + (m["rho"] * m["J"][hinge].T @ m["J"][hinge] if p.M > 0 else 0.0)
    n, na, nU, T = m["n"], A.shape[0], m["nU"], p.T
    K = np.zeros((n + na, n + na))
    K[:n, :n], K[:n, n:], K[n:, :n] = H, A.T, A
    gx = np.zeros(n)
    gx[:nU] = np.asarray(gU, np.float64).T.reshape(-1)
    for t in range(T):
        gx[:nU] += m["F"][t].T @ np.asarray(gS, np.float64)[:, t + 1]
    if p.M > 0:
        gx[nU:] = np.asarray(gD, np.float64).reshape(-1)
    z = np.linalg.lstsq(K.T, np.concatenate([gx, np.zeros(na)]), rcond=None)[0]
    g_theta = backward(p, ref_s, ref_us, gS, gU, gD, tol)
    g_para = np.zeros((3, T + 1))
    for t in range(T):
        g_para[:, t + 1] = p.bk * (m["F"][t] @ z[:nU])  # dF/dpara_s[r,t+1] = -bk F_t[r]'  ->  dL/dpara_s = +bk F_t[r] z
    return g_theta, g_para


def backward_chain(problems, ref_s, ref_us, gS, gU, gD, tol=1e-7):
    """Reference semantics of ``loss.backward()`` through PAN.forward (pan.py:127-147): the K solves are chained through ``nom_s``
    only -- A, B, C (robot.py:272-316: ``torch.Tensor([...])`` of detached numbers), fa, fb (dune.py:78-95 under ``no_grad``, R built
    by ``torch.tensor``) and nom_u carry no gradient.  ``problems`` = the K NrmpProblems in execution order; (gS, gU, gD) = upstream
    gradient of the LAST solve's outputs.  Returns dL/dtheta (7)."""
    total = np.zeros(7)
    gS = np.asarray(gS, np.float64).copy()
    gU = np.asarray(gU, np.float64).copy()
    gD = np.asarray(gD, np.float64).copy()
    for p in reversed(problems):
        g_theta, g_para = backward_full(p, ref_s, ref_us, gS, gU, gD, tol)
        total += g_theta
        gS, gU, gD = g_para, np.zeros_like(gU), np.zeros_like(gD)
    return total


def chain_loss(problems, ref_s, ref_us, theta, wS, wU, wD):
    """L(theta) = <wS, S_K> + <wU, U_K> + <wD, D_K> of the K-solve chain with FROZEN coefficients: solve k uses problems[k]'s
    A, B, C, fa, fb and (theta, para_s = S_{k-1}(theta)) -- the function whose gradient backward_chain states.  For finite
    differences in the tests."""
    S_prev = None
    for k, p in enumerate(problems):
        q = with_theta(p, ref_s, ref_us, theta)
        if S_prev is not None:
            ns = q.nom_s.copy()
            ns[:, 1:] = S_prev[:, 1:]
            q = dataclasses.replace(q, nom_s=ns)
        S, U, D, _ = ipm.solve_ipm(q)
        S_prev = S
    val = float(np.sum(wS * S) + np.sum(wU * U))
    if problems[-1].M > 0:
        val += float(np.sum(wD * D.reshape(-1)))
    return val
