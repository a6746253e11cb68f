"""A/B timing of build variants in ONE process launch per variant (saves gpurun round trips).

    # here (no GPU): build the default library plus variants that differ by -D flags on one translation unit
    python tools/ab_bench.py build  nrmp7:nrmp.cu:-DNB_SOME_FLAG=1  tcx:dune_tc.cu:-DNB_OTHER=2
    # on the GPU machine: time the default and every built variant with bench.py
    python tools/ab_bench.py run --steps 6 --warmup 3

Variants are written to neupan_b200/lib/variants/<name>.so (git-ignored like every built .so; they travel with the snapshot)
and selected through NEUPAN_B200_LIB (neupan_b200/_lib.py).  The default library and its stamp are left untouched.
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
VARDIR = os.path.join(ROOT, "neupan_b200", "lib", "variants")


def build(specs):
    from neupan_b200 import build as nb

    nb.build()  # default library + all default objects
    os.makedirs(VARDIR, exist_ok=True)
    nvcc = nb._nvcc()
    for spec in specs:
        name, tu, *flags = spec.split(":")
        if tu not in nb.UNITS:
            raise SystemExit(f"{tu} is not one of the library's translation units {nb.UNITS}")
        obj = os.path.join(VARDIR, f"{name}_{os.path.splitext(tu)[0]}.o")
        subprocess.run([nvcc, *nb.ARCH, *nb.COMMON, *flags, "-c", os.path.join(nb.CSRC, tu), "-o", obj], check=True)
        objs = [obj if u == tu else nb.obj_path(u) for u in nb.UNITS]
        subprocess.run([nvcc, *nb.ARCH, "-shared", "-o", os.path.join(VARDIR, f"{name}.so"), *objs], check=True)
        print("built", name)


def run(extra):
    libs = [("default", "")] + [(f[:-3], os.path.join(VARDIR, f)) for f in sorted(os.listdir(VARDIR)) if f.endswith(".so")] if os.path.isdir(VARDIR) else [("default", "")]
    for name, path in libs:
        env = dict(os.environ, NEUPAN_B200_LIB=path)
        r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--no-cpu", *extra], env=env, capture_output=True, text=True)
        try:
            d = json.loads(r.stdout.strip().splitlines()[-1])
            print(f"{name:24s} step {d['ms_per_step']:8.3f} ms   DUNE {d['roofline']['kernel_ms']:.3f} ms   {d['value']:.0f} {d['unit']}")
        except Exception:
            print(f"{name:24s} FAILED: {r.stderr.strip().splitlines()[-1] if r.stderr.strip() else r.stdout[-200:]}")


if __name__ == "__main__":
    if len(sys.argv) >= 2 and sys.argv[1] == "build":
        build(sys.argv[2:])
    elif len(sys.argv) >= 2 and sys.argv[1] == "run":
        run(sys.argv[2:])
    else:
        print(__doc__)
