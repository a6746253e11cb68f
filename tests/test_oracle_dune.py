"""Pins oracle/dune.py (the CPU restatement of the DUNE half) against the reference's own code: golden vectors produced by
that code (tests/golden/ref_dune_*.npz, made by make_golden.py; ref_dune_flow.npz, made by make_golden_dune_flow.py) and,
where the reference checkout is present, a check that those vectors are current."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN, weights_path
from oracle import dune as od
from oracle.refload import reference_available

_spec = importlib.util.spec_from_file_location("make_golden_dune_flow", os.path.join(GOLDEN, "make_golden_dune_flow.py"))
mgf = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mgf)


@pytest.mark.parametrize("model", ["diff", "acker", "polygon"])
@pytest.mark.parametrize("case", ["a", "b", "c", "d"])
def test_dune_matches_reference_golden(model, case):
    z = np.load(f"{GOLDEN}/ref_dune_{model}.npz")
    w = od.load_weights(weights_path(model))
    G = torch.from_numpy(z["G"]).float(); h = torch.from_numpy(z["h"]).float()
    nom_s = torch.from_numpy(z[f"{case}_nom_s"]); pts = torch.from_numpy(z[f"{case}_points"])
    vel = z[f"{case}_vel"]; vel = None if vel.size == 0 else torch.from_numpy(vel)
    T = nom_s.shape[1] - 1
    p0, R, pl = od.point_flow(nom_s, pts, vel, T, 0.1, int(z[f"{case}_dune_max_num"]))
    mu, lam, sp, md, _ = od.dune_forward(w, G, h, p0, R, pl, stable=False)
    assert np.array_equal(torch.stack(p0).numpy(), z[f"{case}_p0"])
    assert np.array_equal(torch.stack(R).numpy(), z[f"{case}_R"])
    assert np.array_equal(torch.stack(mu).numpy(), z[f"{case}_mu"])  # bit-for-bit
    assert np.array_equal(torch.stack(lam).numpy(), z[f"{case}_lam"])
    assert np.array_equal(torch.stack(sp).numpy(), z[f"{case}_sorted_points"])
    assert np.float32(md) == z[f"{case}_min_distance"]
    assert np.array_equal(pl[0].numpy(), z[f"{case}_dune_points"])
    # the deterministic (stable) order differs from the reference order only inside exact ties
    mu_s, lam_s, sp_s, _, dist = od.dune_forward(w, G, h, p0, R, pl, stable=True)
    for t in range(T + 1):
        d_ref = od.objective_distance(G, h, mu[t], None if False else (R[t].T @ (sp[t] - nom_s[0:2, t:t + 1])))
        d_stb = od.objective_distance(G, h, mu_s[t], (R[t].T @ (sp_s[t] - nom_s[0:2, t:t + 1])))
        assert torch.equal(d_ref, d_stb)


def test_dune_matches_reference_point_flow_fixture():
    """The reference's own point flow + DUNE (acker checkpoint, 200 moving points; tests/golden/make_golden_dune_flow.py) vs
    oracle/dune.py on the same inputs: bit for bit."""
    z = np.load(f"{GOLDEN}/ref_dune_flow.npz")
    T, dt, n = mgf.T, mgf.DT, mgf.DUNE_MAX_NUM
    nom_s, pts, vel = torch.from_numpy(z["nom_s"]), torch.from_numpy(z["points"]), torch.from_numpy(z["vel"])
    p0, R, pl = od.point_flow(nom_s, pts, vel, T, dt, n)
    mu, lam, sp, md, _ = od.dune_forward(od.load_weights(weights_path("acker")), torch.from_numpy(z["G"]).float(), torch.from_numpy(z["h"]).float(),
                                         p0, R, pl, stable=False)
    assert np.array_equal(torch.stack(mu).numpy(), z["mu"])
    assert np.array_equal(torch.stack(lam).numpy(), z["lam"])
    assert np.array_equal(torch.stack(sp).numpy(), z["sorted_points"])
    assert np.float32(md) == z["min_distance"]


@pytest.mark.skipif(not reference_available(), reason="needs the reference checkout")
def test_dune_matches_live_reference():
    """The fixture above is current: the reference's code reproduces it, and the weights fixture equals its checkpoint."""
    from oracle.refload import REFERENCE_ROOT

    fresh, z = mgf.reference_dune_flow(), np.load(f"{GOLDEN}/ref_dune_flow.npz")
    for k, v in fresh.items():
        assert np.array_equal(np.asarray(v), z[k]), k
    w, wz = od.load_weights(f"{REFERENCE_ROOT}/example/model/acker_robot_default/model_5000.pth"), od.load_weights(weights_path("acker"))
    assert all(torch.equal(w[k], wz[k]) for k in w)
