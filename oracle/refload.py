"""Import the *real* reference (``/root/reference/neupan``) on a machine that lacks its
third-party solver stack, by installing in-memory stub modules for ``cvxpy``,
``cvxpylayers.torch``, ``gctl`` and ``colorama`` before the import.

The torch half of the hot path (ObsPointNet, DUNE.forward, PAN.generate_point_flow /
point_state_transform / stop_criteria, robot.linear_*_model, util.gen_inequal_from_vertex /
downsample_decimation) runs as is.  ``cvxpy`` and ``cvxpylayers.torch`` are replaced by the numeric
shim ``oracle/cvx_shim.py``: the reference's NRMP / robot classes build their program with their own
code and the shim turns it into arrays, evaluates it, certifies optimality and solves it (HiGHS +
active-set polish) -- the solver is NOT ECOS, the program is the reference's.

Used by ``tests/golden/make_golden.py`` (fixture generation) and by the not-gpu tests
that validate ``oracle/dune.py`` against the reference.  /root/reference does not
exist on every machine: everything that calls this must skip when it is absent.
"""
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("NEUPAN_REFERENCE_ROOT", "/root/reference")


def reference_available() -> bool:
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "neupan", "blocks"))


class _Anything:
    """Absorbs any attribute access / call made at import or class-definition time."""

    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        return _Anything()

    def __getattr__(self, name):
        return _Anything()


def _stub(name, **attrs):
    mod = types.ModuleType(name)
    mod.__dict__.update(attrs)

    def _getattr(attr):
        if attr.startswith("__"):  # keep inspect / importlib happy
            raise AttributeError(attr)
        return _Anything

    mod.__getattr__ = _getattr  # type: ignore[attr-defined]
    sys.modules[name] = mod
    return mod


def load_reference():
    """Returns the imported reference package module ``neupan`` (the real code)."""
    if not reference_available():
        raise FileNotFoundError(REFERENCE_ROOT)
    if "neupan" in sys.modules and getattr(sys.modules["neupan"], "__file__", "").startswith(REFERENCE_ROOT):
        return sys.modules["neupan"]
    import torch  # noqa: F401  (import before the stubs exist: torch inspects sys.modules)

    for name in ("gctl", "colorama", "irsim"):
        if name not in sys.modules:
            try:
                __import__(name)
            except Exception:
                _stub(name)
    # cvxpy / cvxpylayers: the numeric shim (oracle/cvx_shim.py) so that the reference's NRMP / robot problem
    # construction runs unmodified; a real installation, if one ever exists, is preferred
    if "cvxpy" not in sys.modules:
        try:
            __import__("cvxpy")
        except Exception:
            from . import cvx_shim

            sys.modules["cvxpy"] = cvx_shim
    if "cvxpylayers" not in sys.modules:
        try:
            __import__("cvxpylayers.torch")
        except Exception:
            from . import cvx_shim

            pkg = types.ModuleType("cvxpylayers")
            sub = types.ModuleType("cvxpylayers.torch")
            sub.CvxpyLayer = cvx_shim.CvxpyLayer
            pkg.torch = sub
            sys.modules["cvxpylayers"], sys.modules["cvxpylayers.torch"] = pkg, sub
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    import neupan as ref  # noqa: E402  (the reference package)

    return ref
