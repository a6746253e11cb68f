"""Behavioural parity of the boundary on the GPU: the edge cases the reference's code paths define
(no points, fewer points than M, ragged batches, decimation, no_obs mode, vector q_s, adjust updates,
stop criterion + its state across calls, capacity growth)."""
import numpy as np
import pytest
import torch

from gpu_helpers import make_pan, record, run_pan, to_cuda
from helpers import CONFIGS, make_inputs, oracle_factory, rel_err
from oracle import pan as op

pytestmark = pytest.mark.gpu
TOL = 1e-4
STOP_SAME_MIN = 0.9  # observed 12/12 in both calls; fraction of envs that must stop at the oracle's iteration count (ratcheted from the observed value)


def _cmp(got, ref, tol=TOL):
    S, U, D, md = got
    So, Uo, Do, mdo, _ = ref
    B = S.shape[0]
    return np.array([max(rel_err(S[b], So[b]), rel_err(U[b], Uo[b]), rel_err(D[b], Do[b, 0]),
                         0.0 if not np.isfinite(mdo[b]) else abs(md[b] - mdo[b])) for b in range(B)])


def test_fewer_points_than_M_and_single_point():
    cfg = CONFIGS["C4"]
    for N in (1, 4, 9):
        inp = make_inputs(cfg, B=3, N=N, scene="obstacles")
        err = _cmp(run_pan(make_pan(cfg, K=1, N=N, max_envs=3), inp), op.run_batch(oracle_factory(cfg, K=1, N=N), inp))
        assert (err < TOL).all(), (N, err)


def test_no_points_and_no_obs_mode():
    cfg = CONFIGS["C2"]
    inp = make_inputs(cfg, B=3)
    inp0 = dict(inp, points=None, velocities=None)
    pan = make_pan(cfg, K=2, max_envs=3)
    t = to_cuda(inp)
    S, U, D = pan(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], None, None)
    So, Uo, Do, mdo, _ = op.run_batch(oracle_factory(cfg, K=2), inp0)
    for b in range(3):
        assert rel_err(S[b].cpu().numpy(), So[b]) < TOL and rel_err(U[b].cpu().numpy(), Uo[b]) < TOL
        assert rel_err(D[b, 0].cpu().numpy(), Do[b, 0]) < TOL
    # no_obs mode (nrmp_max_num == 0, pan.py:85): distance output is None, min_distance is inf
    pan0 = make_pan(cfg, K=2, M=0, max_envs=3)
    S, U, D = pan0(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"])
    assert D is None and pan0.min_distance == float("inf") and pan0.dune_points is None and pan0.nrmp_points is None
    So, Uo, _, _, _ = op.run_batch(oracle_factory(cfg, K=2, M=0), inp)
    for b in range(3):
        assert rel_err(S[b].cpu().numpy(), So[b]) < TOL and rel_err(U[b].cpu().numpy(), Uo[b]) < TOL


def test_ragged_batch_equals_truncated_single_envs():
    cfg = CONFIGS["C4"]
    B, N = 5, 64
    inp = make_inputs(cfg, B=B, N=N, scene="obstacles")
    counts = np.array([64, 10, 0, 33, 3], np.int32)
    pan = make_pan(cfg, K=1, N=N, max_envs=B)
    t = to_cuda(inp)
    S, U, D = pan(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"], num_points=torch.from_numpy(counts).cuda())
    md = pan.min_distance.cpu().numpy()
    for b in range(B):
        one = {k: (None if v is None else v[b:b + 1]) for k, v in inp.items()}
        n = int(counts[b])
        one["points"] = one["points"][:, :, :n] if n else None
        one["velocities"] = one["velocities"][:, :, :n] if n else None
        So, Uo, Do, mdo, _ = op.run_batch(oracle_factory(cfg, K=1, N=max(n, 1)), one)
        assert rel_err(S[b].cpu().numpy(), So[0]) < TOL and rel_err(U[b].cpu().numpy(), Uo[0]) < TOL, b
        assert rel_err(D[b, 0].cpu().numpy(), Do[0, 0]) < TOL
        assert (np.isinf(md[b]) and n == 0) or abs(md[b] - mdo[0]) < TOL
    assert pan.read_selection()["count"].cpu().tolist() == [10, 10, 0, 10, 3]


def test_ragged_batch_with_decimation_equals_single_envs():
    """Ragged batch whose padded width exceeds dune_max_num (ADVICE r1): every environment is decimated over its OWN
    point count, like an unbatched reference call on (2, n_b) points (pan.py:171-174)."""
    cfg = CONFIGS["C4"]
    B, N, DM = 5, 200, 100
    inp = make_inputs(cfg, B=B, N=N, scene="obstacles")
    counts = np.array([200, 150, 100, 37, 101], np.int32)
    pan = make_pan(cfg, K=1, N=N, max_envs=B, dune_max_num=DM)
    t = to_cuda(inp)
    S, U, D = pan(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"], num_points=torch.from_numpy(counts).cuda())
    md = pan.min_distance.cpu().numpy()
    for b in range(B):
        one = {k: (None if v is None else v[b:b + 1]) for k, v in inp.items()}
        n = int(counts[b])
        one["points"], one["velocities"] = one["points"][:, :, :n], one["velocities"][:, :, :n]
        So, Uo, Do, mdo, _ = op.run_batch(oracle_factory(cfg, K=1, N=DM), one)  # the oracle decimates n -> DM like the reference
        assert rel_err(S[b].cpu().numpy(), So[0]) < TOL and rel_err(U[b].cpu().numpy(), Uo[0]) < TOL, b
        assert rel_err(D[b, 0].cpu().numpy(), Do[0, 0]) < TOL and abs(md[b] - mdo[0]) < TOL, b
    assert pan.dune_points.shape[-1] == DM


def test_c4_sweep_1024_envs_status_and_certificate():
    """1024 C4 environments (the range that contains env 934), one PAN iteration: every solve reports status 0 and a random
    subset passes the solver-free KKT certificate of the program built from the GPU's own selection (oracle/nrmp.py)."""
    from helpers import robot_spec
    from oracle import nrmp as onr

    cfg = CONFIGS["C4"]
    B = 1024
    inp = make_inputs(cfg, B=B)
    pan = make_pan(cfg, K=1, max_envs=B)
    S, U, D, md = run_pan(pan, inp)
    st = pan.status.cpu().numpy()
    ipm = pan.ipm_iterations.cpu().numpy()
    record("c4_sweep_1024", status_nonzero=int((st != 0).sum()), ipm_iterations_mean=float(ipm.mean()), ipm_iterations_max=int(ipm.max()),
           ipm_iterations_hist={int(k): int(v) for k, v in zip(*np.unique(ipm, return_counts=True))})
    assert (st == 0).all()
    sel = {k: v.cpu().numpy() for k, v in pan.read_selection().items()}
    _, spec = robot_spec(cfg)
    h = spec.h.reshape(-1).astype(np.float32)
    rng = np.random.default_rng(0)
    worst = 0.0
    for b in [934] + list(rng.choice(B, 23, replace=False)):
        fa = sel["lam"][b, 1:]  # (T, M, 2): list entry t+1 (nrmp.py:244)
        fb = (np.einsum("tmk,tmk->tm", sel["lam"][b, 1:], sel["points"][b, 1:]).astype(np.float32) + (sel["mu"][b, 1:] @ h).astype(np.float32))
        prob = onr.build_problem(spec, onr.Adjust(**cfg.adjust), inp["nom_s"][b], inp["nom_u"][b], inp["ref_s"][b], inp["ref_us"][b], fa, fb, cfg.M)
        res, viol = onr.kkt_certificate(prob, S[b].astype(np.float64), U[b].astype(np.float64), D[b].astype(np.float64), act_tol=2e-5)
        scale = max(1.0, float(np.abs(prob.fb).max() * prob.ro_obs))
        worst = max(worst, res / scale)
        assert viol < 2e-5 and res < 2e-3 * scale, (b, res, viol, scale)
    record("c4_sweep_1024_kkt", worst_relative_stationarity=worst)


def test_decimation_to_dune_max_num():
    cfg = CONFIGS["C1"]
    inp = make_inputs(cfg, B=2, N=300)
    pan = make_pan(cfg, K=1, max_envs=2, dune_max_num=100, N=300)
    got = run_pan(pan, inp)
    ref = op.run_batch(oracle_factory(cfg, K=1, N=100), inp)  # the oracle decimates like pan.py:171-174
    assert (_cmp(got, ref) < TOL).all()
    assert pan.dune_points[0].shape == (2, 100)


def test_vector_qs_and_adjust_update():
    cfg = CONFIGS["C4"]
    inp = make_inputs(cfg, B=3, scene="obstacles")
    adj = dict(cfg.adjust, q_s=[0.5, 0.6, 0.1])
    pan = make_pan(cfg, K=1, max_envs=3, adjust=adj)
    assert (_cmp(run_pan(pan, inp), op.run_batch(oracle_factory(cfg, K=1, adjust=adj), inp)) < TOL).all()
    new = dict(q_s=[1.0, 0.2, 0.3], p_u=0.7, eta=8.0, d_max=0.8, d_min=0.05)
    pan.nrmp_layer.update_adjust_parameters_value(**new)
    pan.reset_state()
    assert (_cmp(run_pan(pan, inp), op.run_batch(oracle_factory(cfg, K=1, adjust=dict(cfg.adjust, **new)), inp)) < TOL).all()
    assert len(pan.nrmp_layer.adjust_parameters) == 5 and pan.nrmp_layer.adjust_parameters[1].item() == pytest.approx(0.7)
    with pytest.raises(ValueError):
        pan.nrmp_layer.update_adjust_parameters_value(q_s=[1.0, 2.0])


def test_stop_criterion_and_state_across_calls():
    """iter_threshold = 0.1 (yaml default): per-env early stop, and PAN.current_nom_values persisting
    from one forward() to the next (pan.py:100-105, 215-243)."""
    cfg = CONFIGS["C5"]  # omni: the iteration contracts, so the criterion actually fires
    B = 12
    inp = make_inputs(cfg, B=B, scene="obstacles")
    pan = make_pan(cfg, K=6, iter_threshold=0.1, max_envs=B)
    mk = oracle_factory(cfg, K=6, iter_threshold=0.1)
    oracles = [mk() for _ in range(B)]
    for call in range(2):
        S, U, D, md = run_pan(pan, inp)
        it = pan.iterations.cpu().numpy()
        same = 0
        for b in range(B):
            o = oracles[b]
            vel = None if inp["velocities"] is None else inp["velocities"][b]
            So, Uo, Do = o.forward(inp["nom_s"][b], inp["nom_u"][b], inp["ref_s"][b], inp["ref_us"][b], inp["points"][b], vel)
            if it[b] == o.iters_run:
                same += 1
        record("stop_criterion", call=call, envs=B, same_iteration_count=same, iterations=[int(v) for v in it])
        assert same >= STOP_SAME_MIN * B, (call, it)
        assert it.min() >= 1 and it.max() <= 6
    assert it.min() < 6  # second call: the stored state lets some envs stop early
    pan.reset_state()
    run_pan(pan, inp)
    assert pan.iterations.cpu().numpy().min() >= 2  # first call after a reset never stops at iteration 1


def test_stop_criterion_as_its_own_kernel_equals_the_fused_one():
    """Batches of >= 256 environments run section 8 of the NRMP kernel (stop criterion, PAN.current_nom_values) as nrmp_stop_kernel
    after the solve; smaller ones keep it inside.  Same arithmetic, same order: trajectories, iteration counts and the state carried
    into the next call are equal bit for bit (NB_NRMP_DEFER_STOP_MIN is read when the handle is created)."""
    import os

    cfg = CONFIGS["C5"]
    inp = make_inputs(cfg, B=300, scene="obstacles")
    outs = []
    for thr_min in ("1000000", "1"):
        os.environ["NB_NRMP_DEFER_STOP_MIN"] = thr_min
        try:
            pan = make_pan(cfg, K=6, iter_threshold=0.1, max_envs=300)
            a = run_pan(pan, inp)
            it1 = pan.iterations.cpu().numpy().copy()
            b = run_pan(pan, inp)  # second call: starts from the state the first one left
            outs.append((a, it1, b, pan.iterations.cpu().numpy().copy()))
        finally:
            del os.environ["NB_NRMP_DEFER_STOP_MIN"]
    (a0, i0, b0, j0), (a1, i1, b1, j1) = outs
    for x, y in zip(a0 + b0, a1 + b1):
        assert np.array_equal(x, y)
    assert np.array_equal(i0, i1) and np.array_equal(j0, j1)
    assert i0.min() < 6  # the criterion did fire


@pytest.mark.parametrize("cname", ["C4", "C5"])
def test_sub_batches_on_internal_streams_equal_one_stream(cname):
    """NB_OPT_OVERLAP (default 2): the batch runs as sub-batches on internal streams -- environments are independent, so trajectories,
    iteration counts and selections equal the single-stream run bit for bit, with the stop criterion switching environments off."""
    cfg = CONFIGS[cname]
    B = 300
    inp = make_inputs(cfg, B=B, scene="obstacles")
    outs = []
    for ov in (1, 2, 4):
        pan = make_pan(cfg, K=4, iter_threshold=0.1, max_envs=B, overlap=ov)
        a = run_pan(pan, inp)
        sel = {k: v.cpu().numpy() for k, v in pan.read_selection().items()}
        outs.append((a, pan.iterations.cpu().numpy().copy(), sel))
    for a, it, sel in outs[1:]:
        for x, y in zip(outs[0][0], a):
            assert np.array_equal(x, y)
        assert np.array_equal(outs[0][1], it)
        for k in ("mu", "lam", "points", "distance", "count"):
            assert np.array_equal(outs[0][2][k], sel[k]), k


def test_host_inputs_with_chunked_upload_equal_device_inputs():
    """nb_pan_forward_h2d / nb_pan_forward_host upload the batch in environment chunks on a copy stream and run the first DUNE pass chunk
    by chunk (batches of >= 64 environments per chunk): same bits as the device-resident call, ragged counts included."""
    cfg = CONFIGS["C2"]
    B = 300
    inp = make_inputs(cfg, B=B, scene="obstacles")
    counts = torch.from_numpy((np.arange(B) * 7 % (cfg.N + 1)).astype(np.int32))
    t = to_cuda(inp)
    pan = make_pan(cfg, K=3, max_envs=B)
    with torch.no_grad():
        ref = pan(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"], num_points=counts.cuda())
        ref = [x.cpu().numpy() for x in ref] + [pan.min_distance.cpu().numpy()]
        pin = {k: (None if v is None else torch.from_numpy(np.ascontiguousarray(v)).pin_memory()) for k, v in inp.items()}
        for mode in ("h2d", "host"):
            out = pan(pin["nom_s"], pin["nom_u"], pin["ref_s"], pin["ref_us"], pin["points"], pin["velocities"], num_points=counts.pin_memory(),
                      device_out=mode == "h2d")
            assert out[0].is_cuda == (mode == "h2d")
            torch.cuda.synchronize()
            got = [x.cpu().numpy() for x in out] + [pan.min_distance.cpu().numpy()]
            for x, y in zip(ref, got):
                assert np.array_equal(x, y), mode


def test_nrmp_warm_start_reaches_the_cold_start_optimum():
    """NB_OPT_NRMP_WARM: iteration 2's solve starts from iteration 1's solution; same optimum to the solver tolerance, fewer
    interior point iterations.  (K = 2: the first solve is cold in both runs, so the inputs of the second are bit-identical.)"""
    for cname, scene in (("C4", "annulus"), ("C4", "obstacles"), ("C2", "obstacles"), ("C5", "obstacles")):
        cfg = CONFIGS[cname]
        B = 32
        inp = make_inputs(cfg, B=B, scene=scene)
        pw, pc = make_pan(cfg, K=2, max_envs=B, nrmp_warm=1), make_pan(cfg, K=2, max_envs=B, nrmp_warm=0)
        a, b = run_pan(pw, inp), run_pan(pc, inp)
        iw, ic = pw.ipm_iterations.cpu().numpy(), pc.ipm_iterations.cpu().numpy()
        err = max(float(np.abs(a[i] - b[i]).max()) for i in range(3))
        record("nrmp_warm_vs_cold", config=cname, scene=scene, max_abs_diff=err, ipm_iterations_warm=float(iw.mean()), ipm_iterations_cold=float(ic.mean()),
               ipm_iterations_warm_max=int(iw.max()), ipm_iterations_cold_max=int(ic.max()))
        assert (pw.status.cpu().numpy() == 0).all() and (pc.status.cpu().numpy() == 0).all()
        assert err < 5e-5, (cname, scene, err)


def test_dmax_equals_dmin_is_a_fixed_distance():
    """d_max == d_min is feasible in the reference's program (D is pinned); ADVICE r1: it used to be reported infeasible."""
    cfg = CONFIGS["C4"]
    adj = dict(cfg.adjust, d_max=0.5, d_min=0.5)
    inp = make_inputs(cfg, B=4, scene="obstacles")
    pan = make_pan(cfg, K=1, max_envs=4, adjust=adj)
    got = run_pan(pan, inp)
    assert (pan.status.cpu().numpy() == 0).all()
    assert np.allclose(got[2], 0.5, atol=1e-7)
    ref = op.run_batch(oracle_factory(cfg, K=1, adjust=adj), inp)  # the interior point oracle has no interior here: HiGHS fallback
    err = _cmp(got, ref)
    record("dmax_equals_dmin", max_err=float(err.max()))
    assert (err < 2 * TOL).all(), err
    bad = make_pan(cfg, K=1, max_envs=4, adjust=dict(cfg.adjust, d_max=0.2, d_min=0.5))
    run_pan(bad, inp)
    assert (bad.status.cpu().numpy() == 4).all()  # d_min > d_max stays infeasible


def test_capacity_growth_and_shape_checks():
    cfg = CONFIGS["C1"]
    pan = make_pan(cfg, K=1, max_envs=1)
    a = run_pan(pan, make_inputs(cfg, B=1))
    b = run_pan(pan, make_inputs(cfg, B=4))  # exceeds max_envs: the native handle is re-created
    assert np.array_equal(a[0][0], b[0][0])
    with pytest.raises(AssertionError):
        pan(torch.zeros(3, 7).cuda(), torch.zeros(2, 10).cuda(), torch.zeros(3, 11).cuda(), torch.zeros(10).cuda())
    assert (pan.status.cpu().numpy() == 0).all()


# build_tc_image (csrc/dune_tc.cu): the warpgroup kernels take the shared-reciprocal tanh only when every LayerNorm output j satisfies
# |2 log2(e) g_j| sqrt(32) + |2 log2(e) beta_j| <= 30 (products rounded to float32 as in the image)
def _tanh_bound(state_dict):
    amax = 0.0
    for i in (1, 6, 11):
        g, be = ((state_dict[f"MLP.{i}.{k}"].double().numpy() * 2.8853900817779268).astype(np.float32).astype(np.float64) for k in ("weight", "bias"))
        amax = max(amax, float((np.abs(g) * np.sqrt(32.0) + np.abs(be)).max()))
    return amax


@pytest.mark.parametrize("dune_kernel,ln_gain", [(4, 1.0), (2, 1.0), (4, 2.5), (2, 2.5)], ids=["4", "2", "4-ln_gain2.5", "2-ln_gain2.5"])
def test_pentagon_robot_five_edges_random_weights(dune_kernel, ln_gain, tmp_path):
    """E = 5 (no shipped checkpoint has E != 4): a randomly initialised ObsPointNet(2, 5) saved in the
    reference's checkpoint format, run through the DUNE kernel and the oracle.  With its LayerNorm gains scaled by 2.5 the tanh
    arguments exceed build_tc_image's bound, so the wgmma kernels take plain reciprocals (dune_tcp_kernel<false>,
    dune_refine_kernel<false>), as for any such checkpoint.  The screening pipeline must give the exact kernel's bits either way."""
    import types

    from neupan_b200 import PAN, ObsPointNet, robot
    from oracle import dune as od, nrmp as onr
    from test_gpu_screen import _assert_equal

    torch.manual_seed(11)
    net = ObsPointNet(2, 5)
    with torch.no_grad():
        for i in (1, 6, 11):
            net.MLP[i].weight.mul_(ln_gain)
    amax = _tanh_bound(net.state_dict())
    assert (amax <= 30.0) == (ln_gain == 1.0), amax  # 16.3 for the default gains of 1, 40.8 scaled
    ck = str(tmp_path / "model_pentagon.pth")
    torch.save(net.state_dict(), ck)
    verts = [[1.2, 0.0], [0.4, 1.1], [-0.9, 0.7], [-0.9, -0.7], [0.4, -1.1]]
    rb = robot(10, 0.1, kinematics="diff", vertices=verts, max_speed=[8, 3], max_acce=[8, 3])
    assert rb.G.shape == (5, 2)
    cfg = CONFIGS["C4"]
    B, N = 4, 96
    inp = make_inputs(cfg, B=B, N=N, scene="obstacles")
    new = lambda dk: PAN(10, 0.1, rb, iter_num=1, dune_max_num=N, nrmp_max_num=10, dune_checkpoint=ck, iter_threshold=0.0,
                         adjust_kwargs=dict(cfg.adjust), max_envs=B, max_points=N, dune_kernel=dk)
    run = lambda pan: (*run_pan(pan, inp), {k: v.cpu().numpy() for k, v in pan.read_selection().items()})
    pan = new(dune_kernel)
    got = run(pan)
    spec = onr.RobotSpec("diff", rb.G, rb.h, rb.max_speed.reshape(-1), rb.max_acce.reshape(-1), 0.1, None)
    w = od.load_weights(ck)
    mk = lambda: op.OraclePAN(spec, w, T=10, iter_num=1, dune_max_num=N, nrmp_max_num=10, iter_threshold=0.0, adjust=onr.Adjust(**cfg.adjust))
    assert (_cmp(got[:4], op.run_batch(mk, inp)) < TOL).all()
    assert got[4]["mu"].shape == (B, 11, 10, 5)
    if dune_kernel == 4:
        _assert_equal(got, run(new(2)))  # selection, mu, lam, distances and the PAN outputs, bit for bit


def test_dune_kernel_option_takes_2_or_4():
    """NB_OPT_DUNE_KERNEL selects the exact kernel on every point (2) or the screening pipeline (4); any other value is refused
    with NB_ERR_INVALID (ValueError in Python) and leaves the handle as it was."""
    from neupan_b200 import _lib

    cfg = CONFIGS["C4"]
    inp = make_inputs(cfg, B=2, scene="obstacles")
    pan = make_pan(cfg, K=1, max_envs=2)
    before = run_pan(pan, inp)
    lib = pan._ensure_handle(2, cfg.N)
    for v in (-1, 0, 1, 3, 5):
        assert lib.nb_pan_set_option(pan._handle, _lib.OPT_DUNE_KERNEL, v) == _lib.NB_ERR_INVALID
        msg = lib.nb_last_error().decode()
        assert "takes 2 (" in msg and "or 4 (" in msg and msg.endswith(f"got {v}"), msg
    after = run_pan(pan, inp)
    for x, y in zip(before, after):
        assert np.array_equal(x, y)
    with pytest.raises(ValueError, match="NB_OPT_DUNE_KERNEL takes 2"):
        run_pan(make_pan(cfg, K=1, max_envs=2, dune_kernel=1), inp)


@pytest.mark.parametrize("T,M", [(12, 8), (20, 12), (6, 3), (10, 1)])
def test_generic_horizon_and_hinge_counts(T, M):
    """Kernel paths that the five BASELINE configs do not reach: NRMP without compile-time (T, M) (generic offsets),
    2T > 32 (two rows of the reduced system per lane), 8 hinge rows per lane, M = 1."""
    import dataclasses

    cfg = dataclasses.replace(CONFIGS["C4"], T=T, M=M, N=96, K=1)
    B = 4
    inp = make_inputs(cfg, B=B, scene="obstacles")
    pan = make_pan(cfg, K=1, max_envs=B)
    got = run_pan(pan, inp)
    ref = op.run_batch(oracle_factory(cfg, K=1), inp)
    err = _cmp(got, ref)
    assert (err < TOL).all(), (T, M, err)
    assert (pan.status.cpu().numpy() == 0).all()
