"""Cost of a 2D Gaussian Splatting step at BASELINE config 2 (1M Gaussians, SH degree 3, 1920x1080).

The training step (forward + backward through autograd, every plane with an upstream gradient) of
GSFunctionSurfel, GSFunctionSurfelGeometry (the 2DGS geometry terms, DESIGN 3.16: gradients on all
six planes) and GSFunctionFusedRGBD on the same scene, and per-kernel CUDA-event times
(gsb_profile_*) of each: the per-Gaussian passes, the binning and the rasterizer pairs.  The three
variants take turns in rounds (their order rotating) so that clock and thermal drift hit all alike;
medians over rounds are reported with the card's name and power limit, read in the same run.  Prints one JSON line.

    python benchmarks/surfel_step.py [--rounds 7] [--steps 10]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from easygaussiansplatting_b200 import _lib  # noqa: E402
from easygaussiansplatting_b200.gsfunction import (Camera, GSFunctionFusedRGBD, GSFunctionSurfel,  # noqa: E402
                                                   GSFunctionSurfelGeometry)
from easygaussiansplatting_b200.scene import synthetic_scene, upstream_gradient  # noqa: E402

N, W, H, SH = 1_000_000, 1920, 1080, 48


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(q.splitlines()[0])
    except Exception:
        power = None
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    lib = _lib.load()
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    kid = {k: names.index(k) for k in ("preprocess_forward", "draw_rgbd", "draw_backward_rgbd", "preprocess_backward",
                                       "surfel_forward", "draw_surfel", "draw_surfel_backward", "surfel_backward",
                                       "draw_2dgs", "draw_2dgs_backward",
                                       "rects+scan", "keys", "sort", "ranges")}
    sc = synthetic_scene(N, W, H, sh_dim=SH, seed=0)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(sc["Rcw"]), T(sc["tcw"]), T(sc["twc"]))
    params = {k: T(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    alphas = T(sc["alphas"][:, None]).requires_grad_()
    us0 = torch.zeros((N, 2), device=dev, requires_grad=True)
    leaves = [params["pws"], params["shs"], alphas, params["scales"], params["rots"]]
    dl = T(upstream_gradient(W, H, 0) * (3.0 * W * H))
    rng = np.random.default_rng(1)
    dld, dla = T(rng.normal(size=(H, W)).astype(np.float32) / 12.0), T(rng.normal(size=(H, W)).astype(np.float32))

    dln = T(rng.normal(size=(3, H, W)).astype(np.float32))
    dlx, dlm = T(rng.normal(size=(H, W)).astype(np.float32)), T(rng.normal(size=(H, W)).astype(np.float32) / 12.0)

    def step_rgbd():
        for p in leaves:
            p.grad = None
        image, depth, alpha, _ = GSFunctionFusedRGBD.apply(params["pws"], params["shs"], alphas, params["scales"],
                                                           params["rots"], us0, cam)
        torch.autograd.backward([image, depth, alpha], [dl, dld, dla])

    def step_surfel():
        for p in leaves:
            p.grad = None
        image, depth, alpha, normal, _ = GSFunctionSurfel.apply(params["pws"], params["shs"], alphas,
                                                                params["scales"], params["rots"], us0, cam)
        torch.autograd.backward([image, depth, alpha, normal], [dl, dld, dla, dln])

    def step_geometry():
        for p in leaves:
            p.grad = None
        image, depth, alpha, normal, dist, med, _ = GSFunctionSurfelGeometry.apply(
            params["pws"], params["shs"], alphas, params["scales"], params["rots"], us0, cam)
        torch.autograd.backward([image, depth, alpha, normal, dist, med], [dl, dld, dla, dln, dlx, dlm])

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    def kernels(fn):
        """per-step ms of each listed kernel over `steps` calls of fn (the binning runs in both)"""
        lib.gsb_profile_enable(1)
        for k in kid.values():  # drop what earlier calls recorded
            lib.gsb_profile_read(k, ctypes.byref(C_d()), ctypes.byref(C_ll()))
        for _ in range(args.steps):
            fn()
        torch.cuda.synchronize()
        lib.gsb_profile_enable(0)
        out = {}
        for name, k in kid.items():
            ms, cnt = C_d(), C_ll()
            lib.gsb_profile_read(k, ctypes.byref(ms), ctypes.byref(cnt))
            if cnt.value:
                out[name] = ms.value / args.steps
        return out

    C_d, C_ll = ctypes.c_double, ctypes.c_longlong
    arms = {"rgbd": step_rgbd, "surfel": step_surfel, "geometry": step_geometry}
    for fn in arms.values():  # warm-up: library load, capacity bounds, allocator
        for _ in range(3):
            fn()
    gpu, power = card()
    res = {m: {"step": []} for m in arms}
    names_ = list(arms)
    for r in range(args.rounds):
        for m in names_[r % 3:] + names_[:r % 3]:
            fn, d = arms[m], res[m]
            d["step"].append(timed(fn))
            for k, v in kernels(fn).items():
                d.setdefault(k, []).append(v)
    med = {m: {k: round(float(np.median(v)), 4) for k, v in d.items()} for m, d in res.items()}
    out = {
        "gpu": gpu, "power_limit_w": power, "config": "N=%d %dx%d SH degree 3" % (N, W, H),
        "rounds": args.rounds, "steps_per_round": args.steps,
        "ms_per_step": med,
        "spread_ms": {m: {k: round(float(np.max(v) - np.min(v)), 4) for k, v in d.items()} for m, d in res.items()},
        "surfel_vs_rgbd_step": round(med["surfel"]["step"] / med["rgbd"]["step"], 4),
        "geometry_vs_surfel_step": round(med["geometry"]["step"] / med["surfel"]["step"], 4),
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
