#!/usr/bin/env python
"""Times the NRMP solve alone (nb_nrmp_forward) at the shapes of a benchmark workload, on obstacle coefficients made once per input set.

    python tools/nrmp_bench.py [--workload C4] [--envs B] [--reps 20] [--warmup 3] [--dump DIR] [--split [--overlap 2]] [--phases]

The inputs are bench.py's (tests/helpers.make_inputs, two sets of distinct environments).  For each set, nb_dune_forward runs once
and the obstacle coefficients of the NRMP program are formed on the device from its selection (nrmp.py:220-261, as
oracle/dune.nrmp_coefficients does): fa = lam rows, fb = lam.p + mu.h, rows beyond the selected count copy row 0.  The timed
launches alternate between the sets with a 256 MiB L2 flush before each, outside the CUDA events.

Prints one JSON line: ms per launch (mean, min, max), mean / max interior point iterations (nb_pan_read_diagnostics), status
count, the card's name, power limit and SM clock.  --dump DIR writes S, U, D, ipm_iters and status of set 0 as DIR/<name>.npy, so
two builds can be compared output for output.  --split adds a second JSON line: torch.profiler's per-kernel device time of a
bench.py-shaped control step (K PAN iterations, two overlapped sub-batches; --overlap 1: one stream, each kernel's time its own) of the same workload.  --phases times a build of the
library with -DNB_NRMP_PHASES=1 instead (made and cached under neupan_b200/lib/phases/ when its sources changed) and adds the mean
clock64() cycles per warp of the setup (per solve) and of the phases (a)-(e) of the interior point iteration (per iteration) to the
line; the timers' atomics lengthen that build's launch a little.
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, plim, sm, smmax = [c.strip() for c in r.stdout.strip().splitlines()[0].split(",")]
        return dict(gpu=name, power_limit=plim, sm_clock=sm, sm_max_clock=smmax)
    except Exception as e:  # noqa: BLE001 -- reported, not fatal
        return dict(gpu=torch.cuda.get_device_name(0), power_limit=None, sm_clock=None, sm_max_clock=None, nvidia_smi=str(e))


PHASES = ("setup", "a_residual_gap", "b_weights_2x2", "c_V_dmma_assembly", "d_cholesky", "e_newton_passes")


def phases_lib():
    """libneupan_b200.so with nrmp.cu compiled with -DNB_NRMP_PHASES=1, rebuilt when the sources change."""
    from neupan_b200 import build as nb

    nb.build()
    out = os.path.join(nb.LIBDIR, "phases")
    lib, stamp = os.path.join(out, "libneupan_b200.so"), os.path.join(out, "build.stamp")
    digest = hashlib.sha256(nb._sources_digest().encode() + b"NB_NRMP_PHASES").hexdigest()
    if os.path.exists(lib) and os.path.exists(stamp) and open(stamp).read().strip() == digest:
        return lib
    os.makedirs(out, exist_ok=True)
    obj = os.path.join(out, "nrmp.o")
    nvcc = nb._nvcc()
    subprocess.run([nvcc, *nb.ARCH, *nb.COMMON, "-DNB_NRMP_PHASES=1", "-c", os.path.join(nb.CSRC, "nrmp.cu"), "-o", obj], check=True)
    subprocess.run([nvcc, *nb.ARCH, "-shared", "-o", lib, *[obj if u == "nrmp.cu" else nb.obj_path(u) for u in nb.UNITS]], check=True)
    with open(stamp, "w") as f:
        f.write(digest)
    return lib


def read_phases(lib, reset):
    from neupan_b200 import _lib

    buf = (C.c_ulonglong * 8)()
    _lib.check(lib.nb_nrmp_read_phases(buf, int(reset)))
    return [int(v) for v in buf]


def coefficients(sel, h, T, M):
    """fa (B,T,M,2), fb (B,T,M) from the selection of list entries t+1 (nrmp.py:220-261)."""
    lam, pts, mu, cnt = sel["lam"][:, 1:], sel["points"][:, 1:], sel["mu"][:, 1:], sel["count"].long()
    B = lam.shape[0]
    m = torch.arange(M, device=lam.device)
    src = torch.where(m[None, :] < cnt[:, None], m[None, :], torch.zeros_like(m)[None, :])  # (B, M): rows >= count copy row 0
    idx = src[:, None, :].expand(B, T, M)
    lam = torch.gather(lam, 2, idx[..., None].expand(B, T, M, 2))
    pts = torch.gather(pts, 2, idx[..., None].expand(B, T, M, 2))
    mu = torch.gather(mu, 2, idx[..., None].expand(B, T, M, mu.shape[-1]))
    fa = lam.contiguous()
    fb = ((lam * pts).sum(-1) + mu @ h).contiguous()
    empty = (cnt == 0)[:, None, None]
    return torch.where(empty[..., None], 0.0, fa).contiguous(), torch.where(empty, 0.0, fb).contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="C4")
    ap.add_argument("--envs", type=int, default=0, help="B (default: the workload's batch)")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dump", default=None, metavar="DIR")
    ap.add_argument("--split", action="store_true", help="also print torch.profiler's per-kernel split of a bench.py-shaped step")
    ap.add_argument("--overlap", type=int, default=2, help="sub-batch streams of the --split step (1: kernels do not overlap)")
    ap.add_argument("--phases", action="store_true", help="time the NB_NRMP_PHASES build and report cycles per phase")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "nrmp_bench.py times the device"
    if args.phases:
        from neupan_b200 import _lib

        _lib.LIB_PATH = phases_lib()  # before the first _lib.load()

    from gpu_helpers import make_pan
    from helpers import CONFIGS, make_inputs
    from neupan_b200 import _lib

    cfg = CONFIGS[args.workload]
    B, T, M = args.envs or cfg.B, cfg.T, cfg.M
    dev = torch.device("cuda", 0)
    pan = make_pan(cfg, K=1, max_envs=B)
    lib = _lib.load()
    h = torch.from_numpy(np.asarray(cfg.make_robot().h, np.float32).reshape(-1)).to(dev)
    p = lambda x: None if x is None else C.c_void_p(x.data_ptr())
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    sets = []
    for s in range(2):
        inp = make_inputs(cfg, B=B, env_offset=s * B)
        d = {k: (None if v is None else torch.from_numpy(v).to(dev)) for k, v in inp.items()}
        with torch.no_grad():
            pan(d["nom_s"], d["nom_u"], d["ref_s"], d["ref_us"], d["points"], d["velocities"])  # handle, settings, first-launch costs
        _lib.check(lib.nb_dune_forward(pan._handle, B, d["points"].shape[-1], p(d["nom_s"]), p(d["points"]), p(d["velocities"]), None, None, st))
        d["fa"], d["fb"] = coefficients(pan.read_selection(), h, T, M)
        d["S"], d["U"] = torch.empty_like(d["nom_s"]), torch.empty_like(d["nom_u"])
        d["D"], d["status"] = torch.empty(B, T, device=dev), torch.empty(B, dtype=torch.int32, device=dev)
        sets.append(d)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def launch(d):
        _lib.check(lib.nb_nrmp_forward(pan._handle, B, p(d["nom_s"]), p(d["nom_u"]), p(d["ref_s"]), p(d["ref_us"]), p(d["fa"]), p(d["fb"]),
                                       p(d["S"]), p(d["U"]), p(d["D"]), p(d["status"]), st))

    for i in range(args.warmup):
        flush.zero_()
        launch(sets[i % 2])
    torch.cuda.synchronize()
    if args.phases:
        lib.nb_nrmp_read_phases.restype, lib.nb_nrmp_read_phases.argtypes = C.c_int, [C.c_void_p, C.c_int]
        read_phases(lib, True)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.reps)]
    iters = []
    for i in range(args.reps):
        flush.zero_()
        ev[i][0].record()
        launch(sets[i % 2])
        ev[i][1].record()
        if i < 2:  # diagnostics of each set (read after its launch, on the same stream)
            it = torch.empty(B, dtype=torch.int32, device=dev)
            _lib.check(lib.nb_pan_read_diagnostics(pan._handle, B, p(it), st))
            iters.append(it)
    torch.cuda.synchronize()
    ms = np.array([a.elapsed_time(b) for a, b in ev])
    it_all = torch.cat(iters).float()
    bad = int(sum(int((d["status"] != 0).sum()) for d in sets))
    line = dict(metric="nb_nrmp_forward ms per launch", workload=f"{args.workload} {cfg.name}", envs=B, T=T, M=M, reps=args.reps, warmup=args.warmup,
                ms_per_launch=float(ms.mean()), ms_min=float(ms.min()), ms_max=float(ms.max()), ipm_iters_mean=float(it_all.mean()),
                ipm_iters_max=int(it_all.max()), envs_with_status=bad, lib=os.path.basename(_lib.LIB_PATH), **gpu_info())
    if args.phases:
        cyc = read_phases(lib, True)
        iters_, solves = max(cyc[6], 1), max(cyc[7], 1)
        line["phase_cycles"] = dict(setup_per_solve=cyc[0] / solves, **{k: cyc[i] / iters_ for i, k in enumerate(PHASES) if i > 0})
        line["phase_cycles"]["iteration_total"] = sum(cyc[1:6]) / iters_
        line["phase_counts"] = dict(solves=cyc[7], iterations=cyc[6])
        line["lib"] = "phases/" + line["lib"]
    print(json.dumps(line), flush=True)

    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
        launch(sets[0])
        it = torch.empty(B, dtype=torch.int32, device=dev)
        _lib.check(lib.nb_pan_read_diagnostics(pan._handle, B, p(it), st))
        torch.cuda.synchronize()
        for name, v in (("S", sets[0]["S"]), ("U", sets[0]["U"]), ("D", sets[0]["D"]), ("ipm_iters", it), ("status", sets[0]["status"])):
            np.save(os.path.join(args.dump, f"{name}.npy"), v.cpu().numpy())
    pan.close()
    del sets

    if args.split:
        split(cfg, B, args, dev)


def split(cfg, B, args, dev):
    """Per-kernel device time of a bench.py-shaped step: K iterations forced, --overlap sub-batches, L2 flushed between steps."""
    from gpu_helpers import make_pan
    from helpers import make_inputs
    from torch.profiler import ProfilerActivity, profile

    pan = make_pan(cfg, K=cfg.K, max_envs=B, overlap=args.overlap)
    inp = make_inputs(cfg, B=B)
    d = {k: (None if v is None else torch.from_numpy(v).to(dev)) for k, v in inp.items()}
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    step = lambda: pan(d["nom_s"], d["nom_u"], d["ref_s"], d["ref_us"], d["points"], d["velocities"])
    steps = max(3, args.reps // 4)
    with torch.no_grad():
        for _ in range(args.warmup):
            flush.zero_()
            step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                flush.zero_()
                step()
            torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t <= 0 or e.key.startswith(("Memset", "Memcpy")) or "elementwise" in e.key:
            continue
        name = e.key.replace("void ", "").split("(")[0]
        per[name] = per.get(name, 0.0) + t / 1e3 / steps
    tot = sum(per.values())
    line = dict(metric="per-kernel device ms per control step (torch.profiler)", workload=f"{args.workload} {cfg.name}: B={B} T={cfg.T} K={cfg.K}, overlap {args.overlap}",
                steps=steps, kernel_ms_per_step=dict(sorted(per.items(), key=lambda kv: -kv[1])), kernel_ms_sum=tot,
                note="the two sub-batches run on two streams, so kernel times overlap and their sum exceeds the step time", **gpu_info())
    print(json.dumps(line), flush=True)
    pan.close()


if __name__ == "__main__":
    main()
