"""Second, independently written float64 solver for the NRMP program (TEST INFRASTRUCTURE).

Condensed form: the states are eliminated through the linearised dynamics
(robot.py:200-221), s_{t+1} = s0_{t+1} + F_t x_U, leaving x = (U (2T), D (T)); the squared hinge
of robot.py:183-198 is lifted with slacks w_tm >= 0, w_tm >= D_t + fb_tm - fa_tm.s_{t+1,xy} that are
eliminated analytically inside every Newton step, so each iteration of the Mehrotra
predictor-corrector primal-dual interior point method factors one dense 3T x 3T SPD matrix.
The iterate is kept strictly primal feasible (all constraints are linear), so only the dual
residual and the complementarity gap have to be driven to zero.

This is also the algorithm the CUDA kernel implements (one warp per environment); the CUDA
code is written from this derivation, and this file is the checker for it -- never the product.
"""
from __future__ import annotations

import numpy as np

from .nrmp import NrmpProblem


def condense(p: NrmpProblem):
    """Returns s0 (T,3) free response, F (T,3,2T) sensitivities ds_{t+1}/dU, column order
    [u_{0,0},u_{1,0},u_{0,1},u_{1,1},...] (time-major)."""
    T = p.T
    s0 = np.zeros((T, 3))
    F = np.zeros((T, 3, 2 * T))
    s_prev = p.nom_s[:, 0].copy()
    F_prev = np.zeros((3, 2 * T))
    for t in range(T):
        s0[t] = p.A[t] @ s_prev + p.C[t]
        F[t] = p.A[t] @ F_prev
        F[t][:, 2 * t:2 * t + 2] += p.B[t]
        s_prev, F_prev = s0[t], F[t]
    return s0, F


def assemble(p: NrmpProblem):
    """The condensed program in matrix form:  min 0.5 x'Px + c'x + (rho/2) sum_k max(0, J_k x + k_k)^2  s.t.  Ab x <= bb,
    x = (U time-major (2T), D (T)).  Returns a dict with P, c, Ab, bb, J, k, rho, n, nU, nD, s0, F, T, M."""
    T, M = p.T, p.M
    nU = 2 * T
    nD = T if M > 0 else 0
    n = nU + nD
    s0, F = condense(p)
    rows_s = 2 if p.omni else 3
    qd = np.array([2 * (p.q[i] ** 2 if i < rows_s else 0.0) + p.bk for i in range(3)])

    # quadratic part 0.5 x^T P x + c^T x
    P = np.zeros((n, n))
    c = np.zeros(n)
    for t in range(T):
        g = np.array([2 * (p.q[i] if i < rows_s else 0.0) * p.gamma_a[i, t + 1] + p.bk * p.nom_s[i, t + 1] for i in range(3)])
        P[:nU, :nU] += F[t].T @ (qd[:, None] * F[t])
        c[:nU] += F[t].T @ (qd * s0[t] - g)
        P[2 * t, 2 * t] += 2 * p.p_u ** 2
        c[2 * t] += -2 * p.p_u * p.gamma_b[t]
    if M > 0:
        c[nU:] = -p.eta

    # linear inequality rows a^T x <= b on x: boxes on U, rates on U, bounds on D
    Ab, bb = [], []

    def row(entries, rhs):
        a = np.zeros(n)
        for j, v in entries:
            a[j] = v
        Ab.append(a); bb.append(rhs)

    for i in range(2):
        sb = p.speed_bound[i]
        if np.isfinite(sb):
            for t in range(T):
                row([(2 * t + i, 1.0)], sb)
                row([(2 * t + i, -1.0)], sb)
        ab = p.acce_bound[i]
        if np.isfinite(ab):
            for t in range(T - 1):
                row([(2 * t + 2 + i, 1.0), (2 * t + i, -1.0)], ab)
                row([(2 * t + 2 + i, -1.0), (2 * t + i, 1.0)], ab)
    for t in range(nD):
        row([(nU + t, 1.0)], p.d_max)
        row([(nU + t, -1.0)], -max(p.d_min, 0.0))
    Ab = np.array(Ab).reshape(-1, n)
    bb = np.array(bb)

    # hinge rows: r_tm(x) = J_tm x + k_tm ; J = e_D - fa.F_xy ; k = fb - fa.s0_xy
    J = np.zeros((T * M, n))
    k = np.zeros(T * M)
    for t in range(T):
        for m in range(M):
            J[t * M + m, :nU] = -(p.fa[t, m] @ F[t][0:2])
            J[t * M + m, nU + t] = 1.0
            k[t * M + m] = p.fb[t, m] - p.fa[t, m] @ s0[t][0:2]
    rho = p.ro_obs

    return dict(P=P, c=c, Ab=Ab, bb=bb, J=J, k=k, rho=rho, n=n, nU=nU, nD=nD, s0=s0, F=F, T=T, M=M)


class IpmFailure(RuntimeError):
    """The interior point iteration could neither converge nor hand back an acceptable iterate."""


def _guarded_cholesky(H):
    """Cholesky with a growing diagonal shift.  Near the end of the iteration the barrier weights
    W = z/s of the active rows reach 1e12+ and H loses definiteness to rounding; a shift of a few
    ulps of its largest diagonal entry restores it without moving the Newton step measurably."""
    try:
        return np.linalg.cholesky(H), 0.0
    except np.linalg.LinAlgError:
        pass
    d = float(np.abs(np.diag(H)).max())
    shift = 1e-15 * d
    for _ in range(12):
        try:
            return np.linalg.cholesky(H + shift * np.eye(H.shape[0])), shift
        except np.linalg.LinAlgError:
            shift *= 10.0
    raise np.linalg.LinAlgError("H not positive definite even with a 1e-3 relative shift")


def solve_ipm(p: NrmpProblem, max_iter: int = 60, tol: float = 1e-11, verbose: bool = False, info: dict | None = None):
    """Returns S, U, D, iterations.  Termination: complementarity gap < tol and dual residual < 100*tol
    *relative to the problem's gradient scale*; an iteration that stalls in rounding noise below the
    acceptance level (gap < 1e-9, relative residual < 1e-8: still 4 orders below the 1e-4 parity budget)
    returns its best iterate; anything else raises IpmFailure (callers fall back to HiGHS)."""
    m_ = assemble(p)
    P, c, Ab, bb, J, k, rho = m_["P"], m_["c"], m_["Ab"], m_["bb"], m_["J"], m_["k"], m_["rho"]
    n, nU, nD, s0, F, T, M = m_["n"], m_["nU"], m_["nD"], m_["s0"], m_["F"], m_["T"], m_["M"]

    # strictly feasible start
    x = np.zeros(n)
    if M > 0:
        x[nU:] = 0.5 * (p.d_max + max(p.d_min, 0.0))
    sb_ = bb - Ab @ x
    if np.any(sb_ <= 0):
        raise ValueError("no strictly feasible start (bounds empty)")
    r = J @ x + k
    w = np.maximum(r, 0.0) + 1.0
    s_w, s_r = w.copy(), w - r
    z_b, z_w, z_r = 1.0 / sb_, 1.0 / s_w, 1.0 / s_r
    m_tot = len(bb) + 2 * T * M

    # gradient scale of the problem: the residual test is relative to it (an env whose cost gradient is
    # O(1e3) cannot reach an absolute 1e-9 in float64 -- C4 env 934, iteration 5, was the counter-example)
    scale = max(1.0, float(np.abs(c).max()), float(rho * np.abs(k).max()) if M > 0 and k.size else 0.0)
    best = None  # (merit, x, it)
    it = 0
    status = "max_iter"
    for it in range(max_iter):
        rd_x = P @ x + c + Ab.T @ z_b + J.T @ z_r
        rd_w = rho * w - z_w - z_r
        gap = (sb_ @ z_b + s_w @ z_w + s_r @ z_r) / max(m_tot, 1)
        res = max(np.abs(rd_x).max(), np.abs(rd_w).max() if M > 0 else 0.0) / scale
        if verbose:
            print(it, gap, res)
        if gap < 1e-9 and res < 1e-8:
            merit = max(gap, res * 1e-1)
            if best is None or merit < best[0]:
                best = (merit, x.copy(), it, z_b.copy(), sb_.copy())
            elif it - best[2] >= 3:  # three iterations without progress below the acceptance level: rounding floor
                status = "stalled"
                break
        if gap < tol and res < tol * 100:
            status = "converged"
            break
        W_b, W_w, W_r = z_b / sb_, z_w / s_w, z_r / s_r
        Hww = rho + W_w + W_r
        omega = W_r * (rho + W_w) / Hww
        H = P + Ab.T @ (W_b[:, None] * Ab) + J.T @ (omega[:, None] * J)
        try:
            Lc, _shift = _guarded_cholesky(H)
        except np.linalg.LinAlgError:
            status = "cholesky"
            break

        def newton(rc_b, rc_w, rc_r):
            v_b, v_w, v_r = rc_b / sb_, rc_w / s_w, rc_r / s_r
            b_x = -rd_x - Ab.T @ v_b - J.T @ v_r
            b_w = -rd_w + v_w + v_r
            rhs = b_x + J.T @ (W_r * b_w / Hww)
            dx = np.linalg.solve(Lc.T, np.linalg.solve(Lc, rhs))
            Jdx = J @ dx
            dw = (b_w + W_r * Jdx) / Hww
            ds_b = -(Ab @ dx)
            ds_w = dw
            ds_r = dw - Jdx
            dz_b = (rc_b - z_b * ds_b) / sb_
            dz_w = (rc_w - z_w * ds_w) / s_w
            dz_r = (rc_r - z_r * ds_r) / s_r
            return dx, dw, (ds_b, ds_w, ds_r), (dz_b, dz_w, dz_r)

        def max_step(v, dv):
            neg = dv < 0
            return min(1.0, float(np.min(-v[neg] / dv[neg]))) if np.any(neg) else 1.0

        # predictor
        dx, dw, ds, dz = newton(-sb_ * z_b, -s_w * z_w, -s_r * z_r)
        a_aff = min(max_step(sb_, ds[0]), max_step(s_w, ds[1]), max_step(s_r, ds[2]),
                    max_step(z_b, dz[0]), max_step(z_w, dz[1]), max_step(z_r, dz[2]))
        gap_aff = ((sb_ + a_aff * ds[0]) @ (z_b + a_aff * dz[0]) + (s_w + a_aff * ds[1]) @ (z_w + a_aff * dz[1])
                   + (s_r + a_aff * ds[2]) @ (z_r + a_aff * dz[2])) / max(m_tot, 1)
        sigma = (gap_aff / gap) ** 3
        # corrector
        dx, dw, ds, dz = newton(-sb_ * z_b + sigma * gap - ds[0] * dz[0],
                                -s_w * z_w + sigma * gap - ds[1] * dz[1],
                                -s_r * z_r + sigma * gap - ds[2] * dz[2])
        a = min(max_step(sb_, ds[0]), max_step(s_w, ds[1]), max_step(s_r, ds[2]),
                max_step(z_b, dz[0]), max_step(z_w, dz[1]), max_step(z_r, dz[2]))
        a = min(1.0, 0.995 * a)
        x = x + a * dx
        w = w + a * dw
        sb_, s_w, s_r = sb_ + a * ds[0], s_w + a * ds[1], s_r + a * ds[2]
        z_b, z_w, z_r = z_b + a * dz[0], z_w + a * dz[1], z_r + a * dz[2]

    if status != "converged":
        if best is None:
            raise IpmFailure(f"interior point method ended with status {status} at iteration {it} (gap {gap:.2e}, rel. residual {res:.2e})")
        x, z_b, sb_ = best[1], best[3], best[4]
    if info is not None:
        # z_b / s_b: multipliers and slacks of the rows Ab x <= bb at the returned iterate
        info.update(status=status, iterations=it, gap=float(gap), residual=float(res), scale=scale, z_b=z_b, s_b=sb_)
    U = x[:nU].reshape(T, 2).T.copy()
    S = np.zeros((3, T + 1))
    S[:, 0] = p.nom_s[:, 0]
    for t in range(T):
        S[:, t + 1] = s0[t] + F[t] @ x[:nU]
    D = x[nU:].reshape(1, T).copy() if M > 0 else None
    return S, U, D, it
