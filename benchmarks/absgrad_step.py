"""Cost of absolute-gradient densification (AbsGS) at BASELINE config 2 (1M Gaussians, SH degree 3,
1920x1080).

Per-kernel CUDA-event times (gsb_profile_*) of the backward rasterizers k_draw_bwd vs
k_draw_bwd_abs and k_draw_bwd_rgbd vs k_draw_bwd_rgbd_abs, and the fused training step (forward +
backward through autograd) of GSFunctionFused without and with `us_abs` (and the same pair for
GSFunctionFusedRGBD).  The variants alternate in rounds so that clock and thermal drift hit them
alike; medians over rounds are reported with the card's name and power limit, read in the same
run.  `abs_over_plain` is k_draw_bwd_abs / k_draw_bwd: the fused statistic is worth having only well
below 2, the cost of a second backward replay.  Prints one JSON line.

    python benchmarks/absgrad_step.py [--rounds 7] [--steps 10]

GSB_LIB=<path> times another build of the library (e.g. one with -DDRAW_BWD_ABS_MINBLOCKS=5).
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
from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused, GSFunctionFusedRGBD  # noqa: E402
from easygaussiansplatting_b200.scene import synthetic_scene, upstream_gradient  # noqa: E402

N, W, H, SH = 1_000_000, 1920, 1080, 48
KERNELS = ("draw_backward", "draw_backward_abs", "draw_backward_rgbd", "draw_backward_rgbd_abs")


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
    kid = {k: names.index(k) for k in KERNELS}
    sc = synthetic_scene(N, W, H, sh_dim=SH, seed=0)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(sc["Rcw"]), T(sc["tcw"]), T(sc["twc"]))
    params = {k: T(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    alphas = T(sc["alphas"][:, None]).requires_grad_()
    us0 = torch.zeros((N, 2), device=dev, requires_grad=True)
    us_abs = torch.zeros((N, 2), device=dev, requires_grad=True)
    leaves = [params["pws"], params["shs"], alphas, params["scales"], params["rots"], us0, us_abs]
    dl = T(upstream_gradient(W, H, 0) * (3.0 * W * H))
    rng = np.random.default_rng(1)
    dld, dla = T(rng.normal(size=(H, W)).astype(np.float32) / 12.0), T(rng.normal(size=(H, W)).astype(np.float32))
    args_map = [params["pws"], params["shs"], alphas, params["scales"], params["rots"], us0, cam]

    def step(rgbd, absgrad):
        def fn():
            for p in leaves:
                p.grad = None
            extra = (None, us_abs) if absgrad else ()
            if rgbd:
                image, depth, alpha, _ = GSFunctionFusedRGBD.apply(*args_map, *extra)
                torch.autograd.backward([image, depth, alpha], [dl, dld, dla])
            else:
                image, _ = GSFunctionFused.apply(*args_map, *extra)
                image.backward(dl)
        fn.__name__ = "step" + ("_rgbd" if rgbd else "") + ("_abs" if absgrad else "")
        return fn

    steps = [step(False, False), step(False, True), step(True, False), step(True, True)]

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    C_d, C_ll = ctypes.c_double, ctypes.c_longlong

    def kernels(fn):
        """per-launch ms of the four backward rasterizers over `steps` calls of fn"""
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
                out[name] = ms.value / cnt.value
        return out

    for fn in steps:  # warm-up: library load, capacity bounds, allocator
        for _ in range(3):
            fn()
    gpu, power = card()
    res = {fn.__name__: [] for fn in steps}
    res.update({k: [] for k in KERNELS})
    for r in range(args.rounds):
        order = steps if r % 2 == 0 else steps[::-1]
        for fn in order:
            res[fn.__name__].append(timed(fn))
            for k, v in kernels(fn).items():
                res[k].append(v)
    med = {k: float(np.median(v)) for k, v in res.items() if v}
    out = {
        "gpu": gpu, "power_limit_w": power, "config": "N=%d %dx%d SH degree 3" % (N, W, H),
        "library": os.path.basename(_lib.LIB_PATH), "rounds": args.rounds, "steps_per_round": args.steps,
        "ms": {k: round(v, 4) for k, v in med.items()},
        "spread_ms": {k: round(float(np.max(v) - np.min(v)), 4) for k, v in res.items() if v},
        "abs_over_plain": {
            "draw_backward": round(med["draw_backward_abs"] / med["draw_backward"], 4),
            "draw_backward_rgbd": round(med["draw_backward_rgbd_abs"] / med["draw_backward_rgbd"], 4),
            "step": round(med["step_abs"] / med["step"], 4),
            "step_rgbd": round(med["step_rgbd_abs"] / med["step_rgbd"], 4),
        },
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
