"""Golden fixtures of the NRMP program as the REFERENCE'S OWN CODE builds and solves it (neupan/blocks/nrmp.py:263-383,
neupan/robot/robot.py:73-236 and neupan/blocks/pan.py executing unmodified; cvxpy / cvxpylayers = oracle/cvx_shim.py):

* per case of CASES: the canonical program the reference built (objective and constraints as arrays), the solution of the
  reference's own ``NRMP.forward`` (float64, before its cast to float32) and its S, U, D;
* the reference's ``generate_parameter_value`` for C1 / C2 / C5;
* the reference's whole ``PAN.forward`` for C1 (K = 2), C2 (K = 3), C5 (K = 2), two environments each.

    python tests/golden/make_golden_refprog.py      # needs the reference checkout; writes tests/golden/ref_program.npz
"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from helpers import CONFIGS, make_inputs, robot_spec, weights_path  # noqa: E402
from oracle import dune as od, refload  # noqa: E402

CASES = [("C1", {}, None), ("C2", {}, None), ("C4", {}, None), ("C5", {}, None),
         ("C4", dict(q_s=[0.5, 1.5, 0.25]), None), ("C2", dict(q_s=[1.0, 0.3, 2.0], p_u=0.7, eta=8.0, d_max=1.5, d_min=0.2), None),
         ("C1", {}, 0), ("C5", dict(q_s=[1.0, 2.0, 3.0]), 0)]
PARAM_CONFIGS = ("C1", "C2", "C5")
PAN_RUNS = (("C1", 2), ("C2", 3), ("C5", 2))
PAN_ENVS = 2


def case_inputs(cname, adjust_over, M, scene="obstacles", env=0):
    """(cfg, adjust, M, one environment's inputs) of a program case; shared by the fixtures and the tests."""
    cfg = CONFIGS[cname]
    adjust = dict(cfg.adjust); adjust.update(adjust_over)
    Mv = cfg.M if M is None else M
    return cfg, adjust, Mv, make_inputs(cfg, B=1, N=min(cfg.N, 120), scene=scene, env_offset=env)


def dune_lists(cfg, inp, b=0):
    """mu / lam / sorted point lists of one environment from the (reference-pinned) DUNE oracle."""
    _, spec = robot_spec(cfg)
    w = od.load_weights(weights_path(cfg.model))
    G, h = torch.from_numpy(spec.G).float(), torch.from_numpy(spec.h.reshape(-1, 1)).float()
    t = lambda a: None if a is None else torch.from_numpy(a[b])
    vel = None if inp["velocities"] is None else t(inp["velocities"])
    p0, R, p = od.point_flow(t(inp["nom_s"]), t(inp["points"]), vel, cfg.T, cfg.dt, cfg.N)
    mu, lam, sp, _, _ = od.dune_forward(w, G, h, p0, R, p)
    return mu, lam, sp, h, spec


def _ref_layer(cfg, adjust, M):
    refload.load_reference()
    from neupan.blocks.nrmp import NRMP
    from neupan.robot import robot as RefRobot

    rb = RefRobot(cfg.T, cfg.dt, **cfg.robot_kwargs)
    return NRMP(cfg.T, cfg.dt, rb, nrmp_max_num=cfg.M if M is None else M, **adjust)


def reference_case(i):
    """The reference's program of CASES[i], its solution and its S, U, D, as arrays under the key prefix case<i>."""
    cname, adjust_over, M = CASES[i]
    cfg, adjust, Mv, inp = case_inputs(cname, adjust_over, M)
    layer = _ref_layer(cfg, adjust, M)
    t = lambda a: torch.from_numpy(a[0])
    args = (t(inp["nom_s"]), t(inp["nom_u"]), t(inp["ref_s"]), t(inp["ref_us"]))
    if Mv > 0:
        mu, lam, sp, _, _ = dune_lists(cfg, inp)
        S, U, D = layer.forward(*args, mu, lam, sp)
    else:
        S, U, D = layer.forward(*args)
    p = f"case{i}"
    out = layer.nrmp_layer.last_canonical.to_arrays(p)
    out.update({f"{p}.x_ref": np.asarray(layer.nrmp_layer.last_x, np.float64), f"{p}.S": S.numpy(), f"{p}.U": U.numpy()})
    if D is not None:  # M = 0: the program has no distance variable
        out[f"{p}.D"] = D.numpy()
    return out


def reference_params(cname):
    """The reference's generate_parameter_value (nrmp.py:152-166, robot.py:239-316) for one environment of cname."""
    cfg, adjust, _, inp = case_inputs(cname, {}, None)
    layer = _ref_layer(cfg, adjust, None)
    t = lambda a: torch.from_numpy(a[0])
    mu, lam, sp, _, _ = dune_lists(cfg, inp)
    vals = layer.generate_parameter_value(t(inp["nom_s"]), t(inp["nom_u"]), t(inp["ref_s"]), t(inp["ref_us"]), mu, lam, sp)
    return {f"params_{cname}.{k}": v.detach().numpy() for k, v in enumerate(vals)}


def pan_inputs(cname):
    cfg = CONFIGS[cname]
    N = min(cfg.N, 150)
    return cfg, N, make_inputs(cfg, B=PAN_ENVS, N=N, scene="obstacles")


def reference_pan(cname, K):
    """The reference's PAN.forward end to end (pan.py:109-147), only the solver swapped."""
    refload.load_reference()
    from neupan.blocks.pan import PAN as RefPAN
    from neupan.robot import robot as RefRobot

    cfg, N, inp = pan_inputs(cname)
    w = od.load_weights(weights_path(cfg.model))
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        ck = os.path.join(tmp, "model.pth")
        torch.save({k: v for k, v in w.items()}, ck)
        for b in range(PAN_ENVS):
            rb = RefRobot(cfg.T, cfg.dt, **cfg.robot_kwargs)
            rp = RefPAN(cfg.T, cfg.dt, rb, iter_num=K, dune_max_num=N, nrmp_max_num=cfg.M, dune_checkpoint=ck, iter_threshold=0.0, adjust_kwargs=dict(cfg.adjust))
            t = lambda a: None if a is None else torch.from_numpy(a[b])
            S, U, D = rp(t(inp["nom_s"]), t(inp["nom_u"]), t(inp["ref_s"]), t(inp["ref_us"]), t(inp["points"]), t(inp["velocities"]))
            p = f"pan_{cname}_{K}_{b}"
            out.update({f"{p}.S": S.detach().numpy(), f"{p}.U": U.detach().numpy(), f"{p}.D": D.detach().numpy(), f"{p}.md": np.float64(rp.min_distance)})
    return out


if __name__ == "__main__":
    out = {}
    for i in range(len(CASES)):
        out.update(reference_case(i))
    for cname in PARAM_CONFIGS:
        out.update(reference_params(cname))
    for cname, K in PAN_RUNS:
        out.update(reference_pan(cname, K))
    np.savez_compressed(os.path.join(HERE, "ref_program.npz"), **out)
