"""Golden outputs of the compile-time NRMP specialisations nrmp_kernel<4, true, 10, 10> (C4 shape) and nrmp_kernel<5, true, 15, 10>
(C5 shape): nb_nrmp_forward on fixed, seeded problems, with every kinematics and bound regimes that make the speed, rate and
distance rows active.  tests/test_gpu_nrmp_bitwise.py requires the kernel to reproduce S, U, D, status and the interior point
iteration counts bit for bit, so a change to the kernel's addressing or loop shapes that alters one rounding shows up there.

    python tests/golden/make_golden_nrmp_bitwise.py [OUT]    # needs a GPU; writes tests/golden/nrmp_bitwise.npz by default

The inputs are stored with the outputs: the obstacle coefficients fa / fb come from the float64 oracle's DUNE selection
(tests/test_oracle_nrmp_shapes.py: build_case), the trajectories from neupan_b200.synth.make_inputs.  The committed
nrmp_bitwise.npz was made on an H100 with the library of commit 832aa61, the build before the fixed-shape iteration of these two
specialisations; it needs no checkout of the reference project.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

SHAPES = ((10, 10), (15, 10))
# None: the shipped bounds; the others: bound regimes of tests/test_oracle_nrmp_shapes.py (finite and infinite boxes mixed)
REGIMES = (None, "tight", "speed_box_and_angular_rate", "angular_box_and_speed_rate")
ENVS = 12  # per case: half `annulus`, half `obstacles`
INPUTS = ("nom_s", "nom_u", "ref_s", "ref_us", "fa", "fb")
OUTPUTS = ("S", "U", "D", "status", "iters")


def case_name(T, M, kin, regime):
    return f"T{T}_M{M}_{kin}_{regime or 'shipped'}"


def cases():
    from test_oracle_nrmp_shapes import KINS

    for T, M in SHAPES:
        for kin in KINS:
            for regime in REGIMES:
                yield T, M, kin, regime


def main():
    from test_gpu_nrmp_shapes import _solve
    from test_oracle_nrmp_shapes import build_case, case_config, case_inputs

    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "nrmp_bitwise.npz")
    out = {}
    for i, (T, M, kin, regime) in enumerate(cases()):
        cfg = case_config(kin, T, M, regime)
        inp = case_inputs(cfg, B=ENVS, env_offset=1000 + 100 * i)
        fa, fb, _ = build_case(cfg, inp)
        res = _solve(cfg, inp, fa, fb)
        name = case_name(T, M, kin, regime)
        for k, v in dict(inp, fa=fa, fb=fb).items():
            if k in INPUTS:
                out[f"{name}.{k}"] = v
        for k in OUTPUTS:
            out[f"{name}.{k}"] = res[k]
        print(name, "status", np.bincount(res["status"]).tolist(), "iters", res["iters"].min(), res["iters"].max())
    np.savez_compressed(out_path, **out)


if __name__ == "__main__":
    main()
