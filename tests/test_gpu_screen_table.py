"""The screen's distance table (NB_OPT_DUNE_SCREEN_TABLE, csrc/dune_table_kernel.cuh): the mma.sync screening pass looks each point's
distance and error radius up in a per-handle table instead of running the fp16 network.  The candidates may differ, the results may
not: the table screen and the network screen give the same PAN outputs and selections bit for bit, and the table stays inside the
handle's bound c_mu, its memory and its build time budget."""
import numpy as np
import pytest

from gpu_helpers import make_pan, record, run_pan
from helpers import CONFIGS, make_inputs

pytestmark = pytest.mark.gpu


def _run(cfg, inp, K, table):
    pan = make_pan(cfg, K=K, max_envs=inp["nom_s"].shape[0], dune_screen_table=table)
    S, U, D, md = run_pan(pan, inp)
    sel = {k: v.cpu().numpy() for k, v in pan.read_selection().items()}
    return (S, U, D, md, sel), pan


@pytest.mark.parametrize("cname", ["C1", "C2", "C3", "C4", "C5"])
@pytest.mark.parametrize("scene", ["annulus", "obstacles"])
def test_table_screen_equals_network_screen_bitwise(cname, scene):
    cfg = CONFIGS[cname]
    inp = make_inputs(cfg, B=12 if cname != "C5" else 6, scene=scene)
    net, _ = _run(cfg, inp, 3, 0)
    tab, pan = _run(cfg, inp, 3, 1)
    for x, y in zip(net[:4], tab[:4]):
        assert np.array_equal(x, y)
    cnt = net[4]["count"]
    assert np.array_equal(cnt, tab[4]["count"])
    live = np.arange(net[4]["distance"].shape[-1])[None, None, :] < cnt[:, None, None]
    for k in ("mu", "lam", "points", "distance"):
        m = live if net[4][k].ndim == 3 else live[..., None]
        assert np.array_equal(np.where(m, net[4][k], 0), np.where(m, tab[4][k], 0)), k
    st, info = pan.screen_stats(), pan.screen_table()
    record("dune_screen_table", config=cname, scene=scene, **st, **{f"table_{k}": v for k, v in info.items()})
    assert info["bytes"] <= 16 << 20 and 0 < info["build_ms"] < 1000
    assert (info["bytes"] > 0) == (2 * info["max_error_ratio"] <= st["c_mu"])  # the table is kept only with a 2x margin to c_mu
    if cfg.model == "diff":  # C1 and the flagship C4 screen with the table
        assert info["bytes"] > 0
    assert st["max_error_ratio"] < st["c_mu"]


def test_network_screen_builds_no_table():
    cfg = CONFIGS["C4"]
    _, pan = _run(cfg, make_inputs(cfg, B=2), 1, 0)
    assert pan.screen_table()["bytes"] == 0
