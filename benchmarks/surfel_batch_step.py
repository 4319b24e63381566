"""Batched 2D Gaussian Splatting (DESIGN 3.25) against the per-view loop it replaces, on one GPU and one
seeded scene.

One training step = forward of C views + backward of a fixed upstream gradient on every plane of every
view, for GSFunctionSurfel (image, depth, alpha, normal) and GSFunctionSurfelGeometry (those and
distortion, median_depth), two ways each:
  batch  GSFunctionSurfelBatch / GSFunctionSurfelGeometryBatch over the C cameras (one per-surfel pass
         each way, one tall frame);
  loop   C calls of GSFunctionSurfel / GSFunctionSurfelGeometry, gradients summed by autograd.
Cases: batch_step.py's, BASELINE config 5 (2M Gaussians, 8 cameras, 1920x1080) and a small-frame case
(1M Gaussians, 16 cameras, 400x300).  The four variants alternate in rounds in one process; medians
of the step time (device synchronise around each step) and the round-to-round spread, then a profiled
run of each for per-kernel times (gsb_profile_*).  Before timing, the batch's frames are compared with
the loop's (bit equality of every plane).  Prints one JSON line per case with the card's name and
power limit read in the same run; writes nothing else.

    python benchmarks/surfel_batch_step.py [--rounds 5] [--steps 5] [--cases config5,small]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from easygaussiansplatting_b200 import _lib  # noqa: E402
from easygaussiansplatting_b200.gsfunction import (Camera, GSFunctionSurfel, GSFunctionSurfelBatch,  # noqa: E402
                                                   GSFunctionSurfelGeometry, GSFunctionSurfelGeometryBatch)
from easygaussiansplatting_b200.scene import ring_camera, synthetic_scene  # noqa: E402

CASES = {"config5": (2_000_000, 8, 1920, 1080), "small": (1_000_000, 16, 400, 300)}
DEV = "cuda:0"


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(q.splitlines()[0])
    except Exception:
        power = None
    return name, power


def setup(N, C, W, H):
    sc = synthetic_scene(N, W, H, sh_dim=48, seed=0)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    cams = []
    for c in range(C):
        R, t, tw = ring_camera(c, C)
        cams.append(Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(R), T(t), T(tw)))
    P = {k: T(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    P["alphas"] = T(sc["alphas"][:, None]).requires_grad_()
    g = torch.Generator(device=DEV).manual_seed(1)
    s = 1.0 / (W * H)
    G = [torch.randn(shape, generator=g, device=DEV) * s
         for shape in ((C, 3, H, W), (C, H, W), (C, H, W), (C, 3, H, W), (C, H, W), (C, H, W))]
    return cams, P, G


def args(P, us):
    return P["pws"], P["shs"], P["alphas"], P["scales"], P["rots"], us


def step_batch(cams, P, G, geo):
    us = torch.zeros((len(cams), P["pws"].shape[0], 2), device=DEV, requires_grad=True)
    if geo:
        out = GSFunctionSurfelGeometryBatch.apply(*args(P, us), cams)
        torch.autograd.backward(out[:6], G)
    else:
        out = GSFunctionSurfelBatch.apply(*args(P, us), cams)
        torch.autograd.backward(out[:4], G[:4])
    return out


def step_loop(cams, P, G, geo):
    N = P["pws"].shape[0]
    outs, grads = [], []
    for c, cam in enumerate(cams):
        us = torch.zeros((N, 2), device=DEV, requires_grad=True)
        fn = GSFunctionSurfelGeometry if geo else GSFunctionSurfel
        out = fn.apply(*args(P, us), cam)
        k = 6 if geo else 4
        outs.append(out[:k])
        grads += [g[c] for g in G[:k]]
    torch.autograd.backward([o for out in outs for o in out], grads)
    return outs


@torch.no_grad()
def frames_equal(cams, P, geo):
    """every plane of the batch's frames against the loop's, bit for bit"""
    N = P["pws"].shape[0]
    us = torch.zeros((len(cams), N, 2), device=DEV)
    fb = (GSFunctionSurfelGeometryBatch if geo else GSFunctionSurfelBatch).apply(*args(P, us), cams)
    fn = GSFunctionSurfelGeometry if geo else GSFunctionSurfel
    for c, cam in enumerate(cams):
        fs = fn.apply(*args(P, us[c]), cam)
        for a, b in zip(fb, fs):
            if not torch.equal(a[c], b):
                return False
    return True


def timed(fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def kernel_times(lib, fn):
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    lib.gsb_profile_enable(1)
    for k in range(len(names)):  # clear
        lib.gsb_profile_read(k, ctypes.byref(ctypes.c_double()), ctypes.byref(ctypes.c_longlong()))
    fn()
    torch.cuda.synchronize()
    out = {}
    for k, n in enumerate(names):
        ms, cnt = ctypes.c_double(), ctypes.c_longlong()
        lib.gsb_profile_read(k, ctypes.byref(ms), ctypes.byref(cnt))
        if cnt.value:
            out[n] = round(ms.value, 4)
    lib.gsb_profile_enable(0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--cases", default="config5,small")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "surfel_batch_step.py measures on the GPU only"
    lib = _lib.load()
    gpu, power = card()
    for case in a.cases.split(","):
        N, C, W, H = CASES[case]
        cams, P, G = setup(N, C, W, H)
        fns = {"surfel_batch": lambda: step_batch(cams, P, G, False),
               "surfel_loop": lambda: step_loop(cams, P, G, False),
               "geometry_batch": lambda: step_batch(cams, P, G, True),
               "geometry_loop": lambda: step_loop(cams, P, G, True)}
        for f in fns.values():  # warm-up: modules, capacity bounds, allocator
            f(); f()
        equal = {"surfel": frames_equal(cams, P, False), "geometry": frames_equal(cams, P, True)}
        t = {k: [] for k in fns}
        for r in range(a.rounds):
            order = list(fns.items())
            order = order[r % len(order):] + order[:r % len(order)]  # rotate: drift hits every variant alike
            for k, f in order:
                t[k].append(timed(f, a.steps))
        med = {k: round(float(np.median(v)), 3) for k, v in t.items()}
        res = {"case": case, "N": N, "C": C, "W": W, "H": H, "gpu": gpu, "power_limit_w": power,
               "frames_bit_equal": equal, "step_ms_median": med,
               "step_ms_spread": {k: [round(min(v), 3), round(max(v), 3)] for k, v in t.items()},
               "loop_over_batch": {g: round(med[g + "_loop"] / med[g + "_batch"], 3) for g in ("surfel", "geometry")},
               "kernel_ms_per_step": {k: kernel_times(lib, f) for k, f in fns.items()}}
        print(json.dumps(res), flush=True)
        del cams, P, G
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
