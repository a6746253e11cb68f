"""A numeric stand-in for ``cvxpy`` + ``cvxpylayers.torch.CvxpyLayer`` (TEST INFRASTRUCTURE).

Purpose: let the reference's own problem-construction code -- ``neupan/blocks/nrmp.py:263-383`` and
``neupan/robot/robot.py:73-236`` -- *execute unmodified* on a machine without cvxpy / cvxpylayers / diffcp /
ECOS, so that the convex program the oracle (``oracle/nrmp.py``, ``oracle/ipm.py``) and the CUDA kernel solve is
pinned to the reference's code and not to a reading of it.  ``oracle/refload.py`` installs this module as
``cvxpy`` and ``cvxpylayers.torch`` before importing ``/root/reference/neupan``.

What it implements (exactly the surface those two files use, nothing more):

* ``Variable`` / ``Parameter`` / constants, ``+ - * @``, ``multiply``, slicing, ``hstack`` / ``vstack``, ``sum``,
  ``.T`` -- lazily, as affine maps  value = A x + b  of the stacked variable vector x once parameter values are known;
* the atoms ``sum_squares``, ``neg``, ``abs``, ``norm`` and the relations ``== <= >=``;
* ``Problem(Minimize | Maximize, constraints)`` with ``is_dcp``; ``canonical(values)`` returns the program as

      min  sum_i c_i |A_i x + b_i|^2  +  sum_j h_j |max(0, -(A_j x + b_j))|^2  +  l'x + const
      s.t. E x = e,   G x <= g   (+ second order cone rows |A x + b| <= t for ``norm`` constraints, evaluation only)

  and offers ``evaluate`` (objective + constraint violations at a point), ``kkt_certificate`` (solver-free optimality
  check: the objective gradient must be a combination of active-constraint normals, multipliers by NNLS) and
  ``solve`` (HiGHS QP on the slack-lifted form, then an exact active-set polish = one linear KKT solve);
* ``CvxpyLayer(problem, parameters, variables)(*tensors, solver_args=...)`` -> tuple of float64 torch tensors.

It is NOT a modelling language: no DCP analysis (``is_dcp`` returns True for the constructs above and raises on
anything else), no cones beyond the evaluation of ``norm``, and the solver behind it is not ECOS -- what ECOS
returns for these programs remains unobservable here (see oracle/__init__.py).
"""
from __future__ import annotations

import numpy as np

__all__ = ["Variable", "Parameter", "Problem", "Minimize", "Maximize", "sum_squares", "neg", "abs", "norm", "multiply", "hstack", "vstack",
           "sum", "CvxpyLayer", "ECOS"]

ECOS = "ECOS"
_builtin_sum, _builtin_abs = sum, abs


def _to_np(v):
    if hasattr(v, "detach"):  # torch tensor
        v = v.detach().cpu().numpy()
    return np.asarray(v, dtype=np.float64)


class _Aff:
    """value = A @ x + b, flattened in C order of `shape`."""

    __slots__ = ("A", "b", "shape")

    def __init__(self, A, b, shape):
        self.A, self.b, self.shape = A, b, tuple(shape)

    @property
    def size(self):
        return int(np.prod(self.shape)) if self.shape else 1

    def broadcast(self, shape):
        shape = tuple(shape)
        if shape == self.shape:
            return self
        idx = np.broadcast_to(np.arange(self.size).reshape(self.shape), shape).reshape(-1)
        return _Aff(self.A[idx], self.b[idx], shape)

    def value(self, x):
        return (self.A @ x + self.b).reshape(self.shape)


class Expr:
    """Lazy expression node: `shape` is known at construction, `_ev(ctx)` yields an _Aff (affine nodes),
    a _Cost (scalar convex nodes) or an atom marker."""

    kind = "affine"

    def __init__(self, shape, ev, kind="affine", args=()):
        self.shape, self._ev, self.kind, self.args = tuple(shape), ev, kind, args

    # ---- structure ------------------------------------------------------------------
    @property
    def T(self):
        if len(self.shape) < 2:
            return self
        perm = np.arange(int(np.prod(self.shape))).reshape(self.shape).T.reshape(-1)
        shp = self.shape[::-1]
        return Expr(shp, lambda c, s=self: (lambda a: _Aff(a.A[perm], a.b[perm], shp))(s._ev(c)), args=(self,))

    def dim(self):
        return len(self.shape)

    def __getitem__(self, key):
        probe = np.arange(int(np.prod(self.shape)) if self.shape else 1).reshape(self.shape)[key]
        idx, shp = np.asarray(probe).reshape(-1), np.asarray(probe).shape
        return Expr(shp, lambda c, s=self: (lambda a: _Aff(a.A[idx], a.b[idx], shp))(s._ev(c)), args=(self,))

    # ---- arithmetic -----------------------------------------------------------------
    def __neg__(self):
        if self.kind == "cost":
            return _scale(self, -1.0)
        return Expr(self.shape, lambda c, s=self: (lambda a: _Aff(-a.A, -a.b, a.shape))(s._ev(c)), args=(self,))

    def __add__(self, other):
        return _add(self, _wrap(other))

    __radd__ = __add__

    def __sub__(self, other):
        return _add(self, -_wrap(other))

    def __rsub__(self, other):
        return _add(_wrap(other), -self)

    def __mul__(self, other):
        return _mul(_wrap(other), self)

    __rmul__ = __mul__

    def __truediv__(self, other):
        return _mul(_wrap(1.0 / float(other)), self)

    def __matmul__(self, other):
        return _matmul(self, _wrap(other))

    def __rmatmul__(self, other):
        return _matmul(_wrap(other), self)

    __array_priority__ = 1000  # numpy defers to the reflected operators above
    __array_ufunc__ = None

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        """torch.Tensor (op) Expr: torch dispatches here instead of trying the reflected operator."""
        name = getattr(func, "__name__", "")
        a, b = (_wrap(args[0]), _wrap(args[1])) if len(args) == 2 else (None, None)
        if name in ("matmul", "__matmul__", "mm"):
            return _matmul(a, b)
        if name in ("mul", "__mul__", "__rmul__", "multiply"):
            return _mul(a, b)
        if name in ("add", "__add__", "__radd__"):
            return _add(a, b)
        if name in ("sub", "__sub__"):
            return _add(a, -b)
        if name == "__rsub__":
            return _add(b, -a)
        return NotImplemented

    # ---- relations ------------------------------------------------------------------
    def __eq__(self, other):  # noqa: D105
        return Constraint("eq", self, _wrap(other))

    def __le__(self, other):
        return Constraint("le", self, _wrap(other))

    def __ge__(self, other):
        return Constraint("le", _wrap(other), self)

    __hash__ = object.__hash__


class _Const(Expr):
    def __init__(self, value):
        v = _to_np(value)
        super().__init__(v.shape, None)
        self._v = v
        self._ev = lambda c: _Aff(np.zeros((v.size, c.n)), v.reshape(-1).copy(), v.shape)
        self.is_const = True


class Parameter(Expr):
    def __init__(self, shape=(), name=None, value=None, nonneg=False, **kw):
        shape = (shape,) if isinstance(shape, int) else tuple(shape)
        super().__init__(shape, None)
        self.name_, self.nonneg = name, nonneg
        self.value = None if value is None else np.broadcast_to(_to_np(value), shape).copy()
        self._ev = self._eval
        self.is_const = True

    def _eval(self, c):
        v = c.values.get(id(self), self.value)
        if v is None:
            raise ValueError(f"parameter {self.name_} has no value")
        v = _to_np(v)
        size = int(np.prod(self.shape)) if self.shape else 1
        v = v.reshape(self.shape) if v.size == size else np.broadcast_to(v, self.shape)
        return _Aff(np.zeros((size, c.n)), np.array(v, np.float64).reshape(-1), self.shape)

    def name(self):
        return self.name_


class Variable(Expr):
    def __init__(self, shape=(), name=None, nonneg=False, **kw):
        shape = (shape,) if isinstance(shape, int) else tuple(shape)
        super().__init__(shape, None)
        self.name_, self.nonneg, self.value = name, nonneg, None
        self._ev = self._eval

    def _eval(self, c):
        off, n = c.offset[id(self)], int(np.prod(self.shape)) if self.shape else 1
        A = np.zeros((n, c.n))
        A[np.arange(n), off + np.arange(n)] = 1.0
        return _Aff(A, np.zeros(n), self.shape)

    def name(self):
        return self.name_


def _wrap(v):
    return v if isinstance(v, Expr) else _Const(v)


def _is_const(e):
    """No variable below this node (parameters and numbers only)."""
    if isinstance(e, Variable):
        return False
    if getattr(e, "is_const", False):
        return True
    return len(e.args) > 0 and all(_is_const(a) for a in e.args)


def _add(a, b):
    if a.kind == "cost" or b.kind == "cost":
        return _cost_add(a, b)
    shp = np.broadcast_shapes(a.shape, b.shape)

    def ev(c):
        x, y = a._ev(c).broadcast(shp), b._ev(c).broadcast(shp)
        return _Aff(x.A + y.A, x.b + y.b, shp)

    return Expr(shp, ev, args=(a, b))


def _mul(k, e):
    """k * e where at least one side is constant; '*' with a scalar side, elementwise otherwise (cvxpy >= 1.1 semantics
    for scalars; matrix '*' is never used by the reference)."""
    if e.kind == "cost" or k.kind == "cost":
        cost, other = (e, k) if e.kind == "cost" else (k, e)
        if not _is_const(other) or int(np.prod(other.shape) if other.shape else 1) != 1:
            raise NotImplementedError("cost * non-scalar")
        return _scale(cost, other)
    return multiply(k, e)


def multiply(k, e):
    k, e = _wrap(k), _wrap(e)
    if not _is_const(k):
        k, e = e, k
    if not _is_const(k):
        raise NotImplementedError("product of two variable expressions is not affine")
    shp = np.broadcast_shapes(k.shape, e.shape)

    def ev(c):
        kv = np.broadcast_to(k._ev(c).b.reshape(k.shape), shp).reshape(-1)
        x = e._ev(c).broadcast(shp)
        return _Aff(kv[:, None] * x.A, kv * x.b, shp)

    return Expr(shp, ev, args=(k, e))


def _matmul(a, b):
    shp = (np.empty(a.shape) @ np.empty(b.shape)).shape
    if _is_const(a):
        def ev(c):
            M = a._ev(c).b.reshape(a.shape)
            x = b._ev(c)
            # out[i, j] = sum_k M[i, k] x[k, j]  (b may be 1-D)
            xs = b.shape if len(b.shape) == 2 else (b.shape[0], 1)
            XA = x.A.reshape(xs[0], xs[1], -1)
            Xb = x.b.reshape(xs)
            M2 = M if M.ndim == 2 else M.reshape(1, -1)
            OA = np.einsum("ik,kjn->ijn", M2, XA)
            Ob = M2 @ Xb
            return _Aff(OA.reshape(-1, OA.shape[-1]), Ob.reshape(-1), shp)
    elif _is_const(b):
        def ev(c):
            M = b._ev(c).b.reshape(b.shape)
            x = a._ev(c)
            xs = a.shape if len(a.shape) == 2 else (1, a.shape[0])
            XA = x.A.reshape(xs[0], xs[1], -1)
            Xb = x.b.reshape(xs)
            M2 = M if M.ndim == 2 else M.reshape(-1, 1)
            OA = np.einsum("ikn,kj->ijn", XA, M2)
            Ob = Xb @ M2
            return _Aff(OA.reshape(-1, OA.shape[-1]), Ob.reshape(-1), shp)
    else:
        raise NotImplementedError("product of two variable expressions is not affine")
    return Expr(shp, ev, args=(a, b))


def _stack(exprs, axis):
    exprs = [_wrap(e) for e in exprs]
    probes, off = [], 0
    for e in exprs:
        n = int(np.prod(e.shape)) if e.shape else 1
        probes.append(np.arange(off, off + n).reshape(e.shape))
        off += n
    lay = np.hstack(probes) if axis == 1 else np.vstack(probes)  # numpy's rules for 1-D operands = cvxpy's
    idx, shp = lay.reshape(-1), lay.shape

    def ev(c):
        parts = [e._ev(c) for e in exprs]
        A = np.concatenate([p.A for p in parts])
        b = np.concatenate([p.b for p in parts])
        return _Aff(A[idx], b[idx], shp)

    return Expr(shp, ev, args=tuple(exprs))


def hstack(exprs):
    return _stack(exprs, 1)


def vstack(exprs):
    return _stack(exprs, 0)


def sum(e, axis=None):  # noqa: A001
    e = _wrap(e)
    if axis is not None:
        raise NotImplementedError
    return Expr((), lambda c: (lambda a: _Aff(a.A.sum(0, keepdims=True), np.array([a.b.sum()]), ()))(e._ev(c)), args=(e,))


# ---- scalar convex costs ----------------------------------------------------------------------
class _Cost:
    """quads: [(coef, _Aff)] coef * |aff|^2 ; hinges: [(coef, _Aff)] coef * |max(0, -aff)|^2 ; lin: _Aff scalar or None."""

    def __init__(self, quads=(), hinges=(), lin=None):
        self.quads, self.hinges, self.lin = list(quads), list(hinges), lin

    def scaled(self, k):
        return _Cost([(k * c, a) for c, a in self.quads], [(k * c, a) for c, a in self.hinges],
                     None if self.lin is None else _Aff(k * self.lin.A, k * self.lin.b, ()))


def _as_cost(e, c):
    v = e._ev(c)
    if isinstance(v, _Cost):
        return v
    if v.size != 1:
        raise ValueError("objective terms must be scalar")
    return _Cost(lin=_Aff(v.A.reshape(1, -1), v.b.reshape(1), ()))


def _cost_add(a, b):
    def ev(c):
        x, y = _as_cost(a, c), _as_cost(b, c)
        lin = x.lin if y.lin is None else y.lin if x.lin is None else _Aff(x.lin.A + y.lin.A, x.lin.b + y.lin.b, ())
        return _Cost(x.quads + y.quads, x.hinges + y.hinges, lin)

    return Expr((), ev, kind="cost", args=(a, b))


def _scale(cost, k):
    k = _wrap(k)

    def ev(c):
        return _as_cost(cost, c).scaled(float(k._ev(c).b.reshape(-1)[0]))

    return Expr((), ev, kind="cost", args=(cost, k))


def neg(e):
    """max(0, -e) elementwise (cvxpy.neg); only meaningful inside sum_squares here."""
    e = _wrap(e)
    return Expr(e.shape, e._ev, kind="negpart", args=(e,))


def abs(e):  # noqa: A001
    e = _wrap(e)
    return Expr(e.shape, e._ev, kind="abs", args=(e,))


def norm(e, p=2):
    e = _wrap(e)
    if p != 2:
        raise NotImplementedError
    return Expr((), e._ev, kind="norm2", args=(e,))


def sum_squares(e):
    e = _wrap(e)
    if e.kind == "negpart":
        return Expr((), lambda c: _Cost(hinges=[(1.0, e._ev(c))]), kind="cost", args=(e,))
    if e.kind != "affine":
        raise NotImplementedError(f"sum_squares of {e.kind}")
    return Expr((), lambda c: _Cost(quads=[(1.0, e._ev(c))]), kind="cost", args=(e,))


# ---- problem ----------------------------------------------------------------------------------
class Constraint:
    def __init__(self, kind, lhs, rhs):
        self.kind, self.lhs, self.rhs = kind, lhs, rhs  # eq: lhs == rhs ; le: lhs <= rhs

    def __bool__(self):
        raise TypeError("a constraint has no truth value")


class Minimize:
    sign = 1.0

    def __init__(self, e):
        self.e = _wrap(e)


class Maximize(Minimize):
    sign = -1.0


class _Ctx:
    def __init__(self, variables, values):
        self.offset, n = {}, 0
        for v in variables:
            self.offset[id(v)] = n
            n += int(np.prod(v.shape)) if v.shape else 1
        self.n, self.values = n, values


def _collect(e, kind, seen, out):
    if id(e) in seen:
        return
    seen.add(id(e))
    if isinstance(e, kind):
        out.append(e)
    for a in e.args:
        _collect(a, kind, seen, out)


class Canonical:
    """The program as arrays (see the module docstring)."""

    def __init__(self, n, quads, hinges, l, const, E, e, G, g, soc, lb):
        self.n, self.quads, self.hinges, self.l, self.const = n, quads, hinges, l, const
        self.E, self.e, self.G, self.g, self.soc, self.lb = E, e, G, g, soc, lb

    # -- storage: the program as a flat dict of arrays (fixtures of programs built by the reference's own code)
    def to_arrays(self, prefix):
        if self.soc:
            raise NotImplementedError("cone rows are not stored")
        out = {f"{prefix}.{k}": np.asarray(v, np.float64) for k, v in dict(l=self.l, const=self.const, E=self.E, e=self.e, G=self.G, g=self.g, lb=self.lb).items()}
        for name, terms in (("quad", self.quads), ("hinge", self.hinges)):
            out[f"{prefix}.{name}_c"] = np.array([c for c, _ in terms], np.float64)
            for j, (_, a) in enumerate(terms):
                out[f"{prefix}.{name}{j}_A"], out[f"{prefix}.{name}{j}_b"] = np.asarray(a.A, np.float64), np.asarray(a.b, np.float64)
        return out

    @classmethod
    def from_arrays(cls, z, prefix):
        g = lambda k: np.asarray(z[f"{prefix}.{k}"])
        terms = lambda name: [(float(c), _Aff(g(f"{name}{j}_A"), g(f"{name}{j}_b"), (len(g(f"{name}{j}_b")),))) for j, c in enumerate(g(f"{name}_c"))]
        l = g("l")
        return cls(len(l), terms("quad"), terms("hinge"), l, float(g("const")), g("E"), g("e"), g("G"), g("g"), [], g("lb"))

    # -- evaluation
    def objective(self, x):
        v = self.const + self.l @ x
        for c, a in self.quads:
            v += c * np.sum((a.A @ x + a.b) ** 2)
        for c, a in self.hinges:
            v += c * np.sum(np.minimum(a.A @ x + a.b, 0.0) ** 2)
        return float(v)

    def gradient(self, x):
        gr = self.l.copy()
        for c, a in self.quads:
            gr += 2 * c * (a.A.T @ (a.A @ x + a.b))
        for c, a in self.hinges:
            gr += 2 * c * (a.A.T @ np.minimum(a.A @ x + a.b, 0.0))
        return gr

    def violation(self, x):
        v = 0.0
        if len(self.e):
            v = max(v, float(np.abs(self.E @ x - self.e).max()))
        if len(self.g):
            v = max(v, float((self.G @ x - self.g).max()))
        for a, t in self.soc:
            v = max(v, float(np.linalg.norm(a.A @ x + a.b) - (t.A @ x + t.b)[0]))
        return max(v, 0.0)

    def kkt_certificate(self, x, act_tol=1e-6):
        """(stationarity residual, primal violation).  Convex program: a feasible x whose gradient is
        -(E' nu + G_act' z), z >= 0, is optimal.  Multipliers by non-negative least squares (nu split in +/-)."""
        from scipy.optimize import nnls

        if self.soc:
            raise NotImplementedError("certificate for cone rows")
        gr = self.gradient(x)
        cols = []
        if len(self.e):
            cols += [self.E.T, -self.E.T]
        if len(self.g):
            act = (self.g - self.G @ x) <= act_tol
            if act.any():
                cols.append(self.G[act].T)
        if not cols:
            return float(np.abs(gr).max()), self.violation(x)
        Aact = np.concatenate(cols, axis=1)
        z, _ = nnls(Aact, -gr, maxiter=50 * Aact.shape[1] + 500)
        return float(np.abs(gr + Aact @ z).max()), self.violation(x)

    # -- solution
    def solve(self, polish=True):
        """HiGHS QP on the lifted form (hinge slacks), then an exact solve on the active set HiGHS found."""
        from scipy.optimize._highspy import _core as hp
        import scipy.sparse as sp

        if self.soc:
            raise NotImplementedError("cone programs are evaluated, not solved, by this shim")
        n = self.n
        hrows = [(c, a) for c, a in self.hinges]
        nw = _builtin_sum(a.size for _, a in hrows)
        N = n + nw
        H = np.zeros((N, N))
        lin = np.zeros(N)
        lin[:n] = self.l
        for c, a in self.quads:
            H[:n, :n] += 2 * c * (a.A.T @ a.A)
            lin[:n] += 2 * c * (a.A.T @ a.b)
        rows, rl, ru = [], [], []
        off = n
        for c, a in hrows:  # w >= -(A x + b), w >= 0, cost c w^2
            for i in range(a.size):
                H[off + i, off + i] = 2 * c
                r = np.zeros(N)
                r[:n] = a.A[i]
                r[off + i] = 1.0
                rows.append(r); rl.append(-a.b[i]); ru.append(hp.kHighsInf)
            off += a.size
        for i in range(len(self.e)):
            r = np.zeros(N); r[:n] = self.E[i]
            rows.append(r); rl.append(self.e[i]); ru.append(self.e[i])
        for i in range(len(self.g)):
            r = np.zeros(N); r[:n] = self.G[i]
            rows.append(r); rl.append(-hp.kHighsInf); ru.append(self.g[i])
        Amat = sp.csc_matrix(np.array(rows).reshape(-1, N))
        lp = hp.HighsLp()
        lp.num_col_, lp.num_row_ = N, Amat.shape[0]
        lb = np.full(N, -hp.kHighsInf); lb[:n] = np.where(np.isfinite(self.lb), self.lb, -hp.kHighsInf); lb[n:] = 0.0
        lp.col_cost_, lp.col_lower_, lp.col_upper_ = lin, lb, np.full(N, hp.kHighsInf)
        lp.row_lower_, lp.row_upper_ = np.array(rl), np.array(ru)
        lp.a_matrix_.format_ = hp.MatrixFormat.kColwise
        lp.a_matrix_.start_, lp.a_matrix_.index_, lp.a_matrix_.value_ = Amat.indptr.astype(np.int32), Amat.indices.astype(np.int32), Amat.data.astype(np.float64)
        model = hp.HighsModel()
        model.lp_ = lp
        Hl = sp.csc_matrix(np.tril(H))
        model.hessian_.dim_, model.hessian_.format_ = N, hp.HessianFormat.kTriangular
        model.hessian_.start_, model.hessian_.index_, model.hessian_.value_ = Hl.indptr.astype(np.int32), Hl.indices.astype(np.int32), Hl.data.astype(np.float64)
        h = hp._Highs()
        h.setOptionValue("output_flag", bool(__import__("os").environ.get("SHIM_VERBOSE")))
        h.setOptionValue("primal_feasibility_tolerance", 1e-8)
        h.setOptionValue("dual_feasibility_tolerance", 1e-8)
        h.passModel(model)
        h.run()
        # kSolveError = HiGHS' own post-check found a residual just above its tolerance (seen: 2.6e-9 vs 1e-9): the point is
        # still the starting point of the polish below, whose result is verified independently
        if h.getModelStatus() not in (hp.HighsModelStatus.kOptimal, hp.HighsModelStatus.kSolveError):
            raise RuntimeError(f"HiGHS status {h.getModelStatus()}")
        x = np.array(h.getSolution().col_value)[:n]
        return self._polish(x) if polish else x

    def _polish(self, x, tol=1e-6, rounds=8):
        """Active-set refinement: with the active inequality rows (incl. variable bounds) held as equalities and the hinge rows
        split into active / inactive, the program is an equality-constrained QP -> one symmetric linear solve.  Accepted only if the
        result is feasible, keeps the hinge pattern and has non-negative multipliers; otherwise the pattern is updated and retried."""
        n = self.n
        G, g = self.G, self.g
        lbrows = [i for i in range(n) if np.isfinite(self.lb[i])]
        if lbrows:
            Gb = np.zeros((len(lbrows), n)); Gb[np.arange(len(lbrows)), lbrows] = -1.0
            G = np.concatenate([G.reshape(-1, n), Gb]); g = np.concatenate([g, -self.lb[lbrows]])
        best = x
        act = (g - G @ x) <= tol
        for _ in range(rounds):
            H = np.zeros((n, n)); q = self.l.copy()
            for c, a in self.quads:
                H += 2 * c * (a.A.T @ a.A); q += 2 * c * (a.A.T @ a.b)
            masks = []
            for c, a in self.hinges:
                m = (a.A @ x + a.b) < 0
                masks.append(m)
                H += 2 * c * (a.A[m].T @ a.A[m]); q += 2 * c * (a.A[m].T @ a.b[m])
            Cm = np.concatenate([self.E.reshape(-1, n), G[act]]); d = np.concatenate([self.e, g[act]])
            k = Cm.shape[0]
            K = np.zeros((n + k, n + k)); K[:n, :n] = H; K[:n, n:] = Cm.T; K[n:, :n] = Cm
            sol = np.linalg.lstsq(K, np.concatenate([-q, d]), rcond=None)[0]
            xn, mult = sol[:n], sol[n + len(self.e):]
            ok = np.all(G @ xn - g <= 1e-9) and np.all(mult >= -1e-9) and all(np.array_equal(m, (a.A @ xn + a.b) < 0) for m, (c, a) in zip(masks, self.hinges))
            if ok:
                return xn
            # update the pattern: drop rows with negative multipliers, add violated rows, re-evaluate hinges at the new point
            new_act = act.copy()
            ai = np.flatnonzero(act)
            new_act[ai[mult < -1e-9]] = False
            viol = (G @ xn - g) > 1e-9
            if viol.any():  # step back to the boundary along x -> xn
                dirn = xn - x
                slack, rate = g - G @ x, G @ dirn
                with np.errstate(divide="ignore", invalid="ignore"):
                    steps = np.where(rate > 1e-14, slack / rate, np.inf)
                a_ = float(np.clip(steps.min(), 0.0, 1.0))
                xn = x + a_ * dirn
                new_act |= (g - G @ xn) <= tol
            act, x = new_act, xn
        return best


class Problem:
    def __init__(self, objective, constraints=()):
        self.objective, self.constraints = objective, list(constraints)
        vs, seen = [], set()
        _collect(objective.e, Variable, seen, vs)
        for c in self.constraints:
            _collect(c.lhs, Variable, seen, vs)
            _collect(c.rhs, Variable, seen, vs)
        self._variables = vs
        ps, seen = [], set()
        _collect(objective.e, Parameter, seen, ps)
        for c in self.constraints:
            _collect(c.lhs, Parameter, seen, ps)
            _collect(c.rhs, Parameter, seen, ps)
        self._parameters = ps
        self.value = None

    def variables(self):
        return list(self._variables)

    def parameters(self):
        return list(self._parameters)

    def is_dcp(self, dpp=False):
        return True  # every construct this shim accepts is DCP (and DPP: parameters enter affinely)

    is_dpp = is_dcp

    def canonical(self, values=None, variables=None) -> Canonical:
        """values: {Parameter: array}; variables: ordering of x (default: discovery order)."""
        variables = list(variables) if variables is not None else self._variables
        extra = [v for v in self._variables if not any(v is w for w in variables)]
        variables = variables + extra
        ctx = _Ctx(variables, {id(k): v for k, v in (values or {}).items()})
        cost = _as_cost(self.objective.e, ctx).scaled(self.objective.sign)
        n = ctx.n
        l = np.zeros(n) if cost.lin is None else cost.lin.A.reshape(-1).copy()
        const = 0.0 if cost.lin is None else float(cost.lin.b[0])
        E, e, G, g, soc = [], [], [], [], []
        for c in self.constraints:
            if c.lhs.kind == "abs":  # |a| <= r
                a, r = c.lhs._ev(ctx), c.rhs._ev(ctx)
                shp = np.broadcast_shapes(a.shape, r.shape)
                a, r = a.broadcast(shp), r.broadcast(shp)
                fin = np.isfinite(r.b)
                G += [a.A[fin] - r.A[fin], -a.A[fin] - r.A[fin]]; g += [r.b[fin] - a.b[fin], r.b[fin] + a.b[fin]]
                continue
            if c.lhs.kind == "norm2":
                soc.append((c.lhs._ev(ctx), c.rhs._ev(ctx)))
                continue
            a, r = c.lhs._ev(ctx), c.rhs._ev(ctx)
            shp = np.broadcast_shapes(a.shape, r.shape)
            a, r = a.broadcast(shp), r.broadcast(shp)
            if c.kind == "eq":
                E.append(a.A - r.A); e.append(r.b - a.b)
            else:
                fin = np.isfinite(r.b - a.b)
                G.append((a.A - r.A)[fin]); g.append((r.b - a.b)[fin])
        cat = lambda rows, width: np.concatenate(rows).reshape(-1, width) if rows else np.zeros((0, width))
        lb = np.full(n, -np.inf)
        for v in variables:
            if getattr(v, "nonneg", False):
                o = ctx.offset[id(v)]
                lb[o:o + (int(np.prod(v.shape)) if v.shape else 1)] = 0.0
        self._ctx = ctx
        return Canonical(n, cost.quads, cost.hinges, l, const, cat(E, n), np.concatenate(e) if e else np.zeros(0), cat(G, n),
                         np.concatenate(g) if g else np.zeros(0), soc, lb)

    def split(self, x, variables=None):
        """x -> list of arrays shaped like the variables."""
        variables = list(variables) if variables is not None else self._variables
        return [x[self._ctx.offset[id(v)]: self._ctx.offset[id(v)] + (int(np.prod(v.shape)) if v.shape else 1)].reshape(v.shape) for v in variables]


class CvxpyLayer:
    """cvxpylayers.torch.CvxpyLayer stand-in: forward only, float64 out."""

    def __init__(self, problem, parameters, variables, **kw):
        self.problem, self.parameters, self.variables = problem, list(parameters), list(variables)
        self.last_canonical = None

    def to(self, *a, **k):
        return self

    def __call__(self, *values, solver_args=None):
        import torch

        if len(values) != len(self.parameters):
            raise ValueError(f"expected {len(self.parameters)} parameter values, got {len(values)}")
        vals = {p: _to_np(v).reshape(p.shape) for p, v in zip(self.parameters, values)}
        can = self.problem.canonical(vals, self.variables)
        x = can.solve()
        self.last_canonical, self.last_x = can, x
        return tuple(torch.from_numpy(a.copy()) for a in self.problem.split(x, self.variables))
