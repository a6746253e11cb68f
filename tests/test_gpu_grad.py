"""Differentiable NRMP (SURVEY 8f row 3; LON, example/LON/LON_corridor.py:94 `loss.backward()`): the gradients that
``loss.backward()`` delivers to NRMP.adjust_parameters through neupan_b200.PAN (native adjoint solves, nb_pan_backward) against
the float64 oracle ``oracle/nrmp_grad.backward_chain`` -- itself validated against finite differences
(tests/test_oracle_nrmp_grad.py).  Tolerance: 1e-3 of the gradient's scale, every environment (the
oracle differentiates the exact active-set system, the kernel the barrier system with capped weights -- independent formulations)."""
import numpy as np
import pytest
import torch

from gpu_helpers import make_pan, record, to_cuda
from helpers import CONFIGS, make_inputs, oracle_factory
from oracle import nrmp_grad as og

pytestmark = pytest.mark.gpu


def _oracle_chain(cfg, inp, b, K, N, adjust=None):
    pan = oracle_factory(cfg, K=K, N=N, adjust=adjust)()
    probs, orig = [], pan._solve
    pan._solve = lambda prob: (probs.append(prob), orig(prob))[1]
    vel = None if inp["velocities"] is None else inp["velocities"][b]
    pan.forward(inp["nom_s"][b], inp["nom_u"][b], inp["ref_s"][b], inp["ref_us"][b], inp["points"][b], vel)
    ref_s, ref_us = inp["ref_s"][b].astype(np.float64), inp["ref_us"][b].astype(np.float64)
    return [og.with_theta(p, ref_s, ref_us, og.theta_of(p)) for p in probs], ref_s, ref_us


@pytest.mark.parametrize("cname,K", [("C4", 2), ("C1", 2), ("C2", 2), ("C5", 2), ("C4", 4)])
def test_backward_matches_oracle_chain(cname, K):
    cfg = CONFIGS[cname]
    B, N = 6, 80
    inp = make_inputs(cfg, B=B, N=N, scene="obstacles")
    pan = make_pan(cfg, K=K, N=N, max_envs=B)
    t = to_cuda(inp)
    rng = np.random.default_rng(7)
    wS, wU, wD = rng.normal(size=(B, 3, cfg.T + 1)), rng.normal(size=(B, 2, cfg.T)), rng.normal(size=(B, 1, cfg.T))
    wS[:, :, 0] = 0.0
    S, U, D = pan(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"])
    assert S.requires_grad and U.requires_grad and D.requires_grad
    c = lambda a: torch.from_numpy(a).float().cuda()
    loss = (S * c(wS)).sum() + (U * c(wU)).sum() + (D * c(wD)).sum()
    loss.backward()
    per_env = pan.last_grad_theta.cpu().numpy().astype(np.float64)
    want = np.zeros((B, 7))
    for b in range(B):
        probs, ref_s, ref_us = _oracle_chain(cfg, inp, b, K, N)
        want[b] = og.backward_chain(probs, ref_s, ref_us, wS[b], wU[b], wD[b, 0])
    err = np.abs(per_env - want).max(axis=1) / np.maximum(1.0, np.abs(want).max(axis=1))
    ok = err < 1e-3
    record("nrmp_backward", config=cname, K=K, envs=B, within_tol=int(ok.sum()), max_rel_err=float(err.max()), median_rel_err=float(np.median(err)),
           grad_scale=float(np.abs(want).max()))
    assert ok.all(), (err, per_env, want)
    leaves = pan.nrmp_layer.adjust_parameters
    got = np.array([leaves[0].grad.item(), leaves[1].grad.item(), leaves[2].grad.item(), leaves[3].grad.item(), leaves[4].grad.item()])
    tot = per_env.sum(0)
    assert np.allclose(got, [tot[0:3].sum(), tot[3], tot[4], tot[5], tot[6]], rtol=1e-5, atol=1e-5)  # scalar q_s: sum of its three entries
    assert np.abs(want).max() > 1e-3  # not a trivially zero gradient


def test_backward_vector_qs_host_tensors_and_unbatched():
    cfg = CONFIGS["C4"]
    adj = dict(cfg.adjust, q_s=[0.5, 0.8, 0.2])
    inp = make_inputs(cfg, B=1, N=60, scene="obstacles")
    pan = make_pan(cfg, K=2, N=60, max_envs=1, adjust=adj)
    h = {k: (None if v is None else torch.from_numpy(v[0])) for k, v in inp.items()}  # unbatched CPU tensors, like neupan.forward
    S, U, D = pan(h["nom_s"], h["nom_u"], h["ref_s"], h["ref_us"], h["points"], h["velocities"])
    assert S.device.type == "cpu" and S.shape == (3, cfg.T + 1) and D.shape == (1, cfg.T)
    rng = np.random.default_rng(3)
    wS, wU, wD = rng.normal(size=(3, cfg.T + 1)), rng.normal(size=(2, cfg.T)), rng.normal(size=(1, cfg.T))
    wS[:, 0] = 0.0
    loss = (S * torch.from_numpy(wS).float()).sum() + (U * torch.from_numpy(wU).float()).sum() + (D * torch.from_numpy(wD).float()).sum()
    loss.backward()
    probs, ref_s, ref_us = _oracle_chain(cfg, inp, 0, 2, 60, adjust=adj)
    want = og.backward_chain(probs, ref_s, ref_us, wS, wU, wD[0])
    q_grad = pan.nrmp_layer.adjust_parameters[0].grad.numpy().reshape(-1)
    assert q_grad.shape == (3,)
    got = np.concatenate([q_grad, [pan.nrmp_layer.adjust_parameters[i].grad.item() for i in range(1, 5)]])
    err = np.abs(got - want).max() / max(1.0, np.abs(want).max())
    record("nrmp_backward_vector_qs_host", rel_err=float(err))
    assert err < 2e-3, (got, want)


def test_no_grad_and_non_leaf_paths():
    cfg = CONFIGS["C1"]
    inp = make_inputs(cfg, B=2, scene="obstacles")
    pan = make_pan(cfg, K=2, max_envs=2)
    t = to_cuda(inp)
    with torch.no_grad():
        S0, U0, D0 = pan(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"])
    assert not S0.requires_grad
    S1, U1, D1 = pan(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"])
    assert S1.requires_grad
    # differentiable mode only adds the adjoint record: the solution is the same program's optimum
    assert torch.allclose(S0, S1.detach(), atol=2e-6) and torch.allclose(U0, U1.detach(), atol=2e-6)
    stale = S1.sum()
    pan(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"])
    with pytest.raises(RuntimeError):
        stale.backward()  # the adjoint records belong to the latest forward


def test_lon_style_tuning_step_reduces_the_loss():
    """example/LON/LON_corridor.py in miniature: Adam on (p_u, eta, d_max) with the 'stuck' loss 50 + sum(distance)."""
    cfg = CONFIGS["C1"]
    inp = make_inputs(cfg, B=4, scene="obstacles")
    pan = make_pan(cfg, K=2, max_envs=4)
    t = to_cuda(inp)
    q_s, p_u, eta, d_max, d_min = pan.nrmp_layer.adjust_parameters
    opt = torch.optim.Adam([p_u, eta, d_max], lr=5e-2)
    losses = []
    for _ in range(6):
        opt.zero_grad()
        pan.reset_state()
        S, U, D = pan(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"])
        loss = 50 + torch.sum(D)
        loss.backward()
        opt.step()
        pan.nrmp_layer.version += 1  # the leaves changed in place: push the new values to the device
        losses.append(float(loss))
    record("lon_style_tuning", losses=losses, d_max=float(d_max), eta=float(eta))
    assert losses[-1] < losses[0] - 1e-3
