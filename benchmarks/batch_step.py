"""Batched rendering (DESIGN 3.21) against the per-view loops it replaces, on one GPU and one seeded scene.

One training step = forward of C views + backward of a fixed upstream gradient per view, three ways:
  batch  GSFunctionFusedBatch over the C cameras (one per-Gaussian pass each way, one tall frame);
  loop   C calls of GSFunctionFused, gradients summed by autograd;
  multi  parallel.MultiViewStep (world 1): render / backward per view, one factorised reduce.
Cases: BASELINE config 5 (2M Gaussians, 8 cameras, 1920x1080) and a small-frame case (1M Gaussians,
16 cameras, 400x300), where one launch over C*T tiles fills more of the 132 SMs than C launches over T.
The three alternate in rounds in one process; medians of the step time (device synchronise around each
step), then a profiled run of each for per-kernel times (gsb_profile_*).  Prints one JSON line per case
with the card's name and power limit read in the same run; writes nothing else.

    python benchmarks/batch_step.py [--rounds 5] [--steps 5] [--cases config5,small]
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
from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused, GSFunctionFusedBatch  # noqa: E402
from easygaussiansplatting_b200.parallel import MultiViewStep  # noqa: E402
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
    G = torch.randn((C, 3, H, W), generator=g, device=DEV) / (3.0 * W * H)
    return cams, P, G


def step_batch(cams, P, G):
    N = P["pws"].shape[0]
    us = torch.zeros((len(cams), N, 2), device=DEV, requires_grad=True)
    img, _ = GSFunctionFusedBatch.apply(P["pws"], P["shs"], P["alphas"], P["scales"], P["rots"], us, cams)
    img.backward(G)


def step_loop(cams, P, G):
    N = P["pws"].shape[0]
    loss = 0.0
    for c, cam in enumerate(cams):
        us = torch.zeros((N, 2), device=DEV, requires_grad=True)
        img, _ = GSFunctionFused.apply(P["pws"], P["shs"], P["alphas"], P["scales"], P["rots"], us, cam)
        loss = loss + (img * G[c]).sum()
    loss.backward()


def make_multi(P):
    return MultiViewStep(P["pws"].detach(), P["rots"].detach(), P["scales"].detach(), P["shs"].detach(),
                         P["alphas"].detach())


def step_multi(mv, cams, G):
    for c, cam in enumerate(cams):
        _, ctx = mv.render(cam)
        mv.backward(ctx, G[c], last=c == len(cams) - 1)
    mv.reduce()


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
    assert torch.cuda.is_available(), "batch_step.py measures on the GPU only"
    lib = _lib.load()
    gpu, power = card()
    for case in a.cases.split(","):
        N, C, W, H = CASES[case]
        cams, P, G = setup(N, C, W, H)
        mv = make_multi(P)
        fns = {"batch": lambda: step_batch(cams, P, G), "loop": lambda: step_loop(cams, P, G),
               "multi": lambda: step_multi(mv, cams, G)}
        for f in fns.values():  # warm-up: modules, capacity bounds, allocator
            f(); f()
        t = {k: [] for k in fns}
        for _ in range(a.rounds):
            for k, f in fns.items():
                t[k].append(timed(f, a.steps))
        res = {"case": case, "N": N, "C": C, "W": W, "H": H, "gpu": gpu, "power_limit_w": power,
               "step_ms_median": {k: round(float(np.median(v)), 3) for k, v in t.items()},
               "step_ms_spread": {k: [round(min(v), 3), round(max(v), 3)] for k, v in t.items()},
               "kernel_ms_per_step": {k: kernel_times(lib, f) for k, f in fns.items()}}
        print(json.dumps(res), flush=True)
        del cams, P, G, mv
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
