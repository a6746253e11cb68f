"""Helpers for the -m gpu parity tests: build a product PAN for a workload config."""
import numpy as np
import torch

from helpers import CONFIGS, weights_path
from neupan_b200 import PAN


def make_pan(cfg, K=None, iter_threshold=0.0, N=None, adjust=None, M=None, max_envs=1, dune_max_num=None, dune_kernel=4, overlap=1, nrmp_warm=0, **pan_kw):
    rb = cfg.make_robot()
    return PAN(cfg.T, cfg.dt, rb, iter_num=cfg.K if K is None else K, dune_max_num=(cfg.N if N is None else N) if dune_max_num is None else dune_max_num,
               nrmp_max_num=cfg.M if M is None else M, dune_checkpoint=weights_path(cfg.model), iter_threshold=iter_threshold,
               adjust_kwargs=dict(adjust or cfg.adjust), max_envs=max_envs, max_points=cfg.N if N is None else N, dune_kernel=dune_kernel, overlap=overlap, nrmp_warm=nrmp_warm, **pan_kw)


def to_cuda(inp):
    return {k: (None if v is None else torch.from_numpy(np.ascontiguousarray(v)).cuda()) for k, v in inp.items()}


def run_pan(pan, inp, cuda=True):
    t = to_cuda(inp) if cuda else {k: (None if v is None else torch.from_numpy(v)) for k, v in inp.items()}
    with torch.no_grad():  # inference: with autograd recording, PAN runs in differentiable mode (tests/test_gpu_grad.py)
        S, U, D = pan(t["nom_s"], t["nom_u"], t["ref_s"], t["ref_us"], t["points"], t["velocities"])
    return S.cpu().numpy(), U.cpu().numpy(), D.cpu().numpy()[:, 0], pan.min_distance.cpu().numpy()


def record(name: str, **values):
    """Observed parity margins (pass fractions, max errors) of a -m gpu run, printed as one `OBSERVED` JSON line so that the
    thresholds in the tests can be ratcheted to what is observed (pytest -s shows them)."""
    import json

    line = json.dumps(dict(test=name, **{k: (float(v) if isinstance(v, (int, float, np.floating, np.integer)) else v) for k, v in values.items()}))
    print("OBSERVED", line)
