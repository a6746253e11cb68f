"""Golden fixture of the REFERENCE'S OWN DUNE on the reference's own point flow: ``PAN.generate_point_flow`` (pan.py:150-212)
followed by ``DUNE.forward`` (dune.py:58-127) of the acker checkpoint, for one seeded scene of 200 moving points.

    python tests/golden/make_golden_dune_flow.py      # needs the reference checkout; writes tests/golden/ref_dune_flow.npz
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.refload import REFERENCE_ROOT, load_reference  # noqa: E402

T, DT, DUNE_MAX_NUM = 10, 0.1, 80


def scene():
    g = torch.Generator().manual_seed(3)
    nom_s = torch.randn(3, T + 1, generator=g); pts = 6 * torch.randn(2, 200, generator=g); vel = torch.randn(2, 200, generator=g)
    return nom_s, pts, vel


def reference_dune_flow():
    """Inputs, robot geometry and what the reference's point flow + DUNE return for scene()."""
    load_reference()
    from neupan.blocks import DUNE, PAN
    from neupan.robot import robot as RefRobot

    rr = RefRobot(T, DT, kinematics="acker", length=4.6, width=1.6, wheelbase=3)
    dune = DUNE(T, f"{REFERENCE_ROOT}/example/model/acker_robot_default/model_5000.pth", rr, DUNE_MAX_NUM, {})
    fake = types.SimpleNamespace(T=T, dt=DT, dune_max_num=DUNE_MAX_NUM, printed=True, print_once=lambda *_: None)
    fake.point_state_transform = types.MethodType(PAN.point_state_transform, fake)
    nom_s, pts, vel = scene()
    pf, Rl, pl = PAN.generate_point_flow(fake, nom_s, pts, vel)
    mu, lam, sp = dune(pf, Rl, pl)
    return dict(nom_s=nom_s.numpy(), points=pts.numpy(), vel=vel.numpy(), G=np.asarray(rr.G), h=np.asarray(rr.h),
                mu=torch.stack(mu).numpy(), lam=torch.stack(lam).numpy(), sorted_points=torch.stack(sp).numpy(),
                min_distance=np.float32(dune.min_distance))


if __name__ == "__main__":
    np.savez_compressed(os.path.join(HERE, "ref_dune_flow.npz"), **reference_dune_flow())
