"""Cost of the camera gradient at BASELINE config 2 (1M Gaussians, SH degree 3, 1920x1080).

The fused training step (forward + backward through autograd) in three forms, each as RGB and
RGB-D: without the pose (GSFunctionFused / GSFunctionFusedRGBD), with the pose and every Gaussian
parameter (GSFunctionFused[RGBD]Pose, camera and map require grad), and pose only (only the
camera requires grad: the frozen-map tracking step).  Besides the step time, the per-launch
CUDA-event time of the `preprocess_backward` profile scope, which covers the per-Gaussian
backward and, with the pose, the partial-row reduction.  The six variants alternate in rounds
(rotated order) so that clock and thermal drift hit all alike; medians over rounds are reported
with the card's name and power limit, read in the same run.  Prints one JSON line.

    python benchmarks/pose_step.py [--rounds 7] [--steps 10]
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
from easygaussiansplatting_b200.gsfunction import (Camera, GSFunctionFused, GSFunctionFusedPose,  # noqa: E402
                                                   GSFunctionFusedRGBD, GSFunctionFusedRGBDPose)
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
    kpre = names.index("preprocess_backward")
    sc = synthetic_scene(N, W, H, sh_dim=SH, seed=0)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    # a general pose, so every camera term is live
    a = 0.05
    Rcw = T(np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]], np.float32))
    tcw = T(np.array([0.02, -0.01, 0.05], np.float32))
    twc = -(Rcw.t() @ tcw)
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], Rcw, tcw, twc)
    params = {k: T(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    alphas = T(sc["alphas"][:, None]).requires_grad_()
    us0 = torch.zeros((N, 2), device=dev, requires_grad=True)
    leaves = [params["pws"], params["shs"], alphas, params["scales"], params["rots"], us0]
    frozen = [x.detach() for x in leaves]
    pose = [x.clone().requires_grad_() for x in (Rcw, tcw, twc)]
    dl = T(upstream_gradient(W, H, 0) * (3.0 * W * H))
    rng = np.random.default_rng(1)
    dld, dla = T(rng.normal(size=(H, W)).astype(np.float32) / 12.0), T(rng.normal(size=(H, W)).astype(np.float32))

    def step(rgbd, mode):
        for p in leaves + pose:
            p.grad = None
        g = frozen if mode == "pose_only" else leaves
        if mode == "no_pose":
            F = GSFunctionFusedRGBD if rgbd else GSFunctionFused
            out = F.apply(*g, cam)
        else:
            F = GSFunctionFusedRGBDPose if rgbd else GSFunctionFusedPose
            out = F.apply(*g, *pose, cam)
        if rgbd:
            torch.autograd.backward(list(out[:3]), [dl, dld, dla])
        else:
            out[0].backward(dl)

    variants = {("rgbd_" if r else "rgb_") + m: (lambda r=r, m=m: step(r, m))
                for r in (False, True) for m in ("no_pose", "pose_all", "pose_only")}

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

    def pre_bwd(fn):
        """per-launch ms of the preprocess_backward scope over `steps` calls of fn"""
        lib.gsb_profile_enable(1)
        lib.gsb_profile_read(kpre, ctypes.byref(C_d()), ctypes.byref(C_ll()))  # drop earlier records
        for _ in range(args.steps):
            fn()
        torch.cuda.synchronize()
        lib.gsb_profile_enable(0)
        ms, cnt = C_d(), C_ll()
        lib.gsb_profile_read(kpre, ctypes.byref(ms), ctypes.byref(cnt))
        return ms.value / cnt.value

    for fn in variants.values():  # warm-up: library load, capacity bounds, allocator
        for _ in range(3):
            fn()
    gpu, power = card()
    keys = list(variants)
    step_ms = {k: [] for k in keys}
    pre_ms = {k: [] for k in keys}
    for r in range(args.rounds):
        for k in keys[r % len(keys):] + keys[:r % len(keys)]:
            step_ms[k].append(timed(variants[k]))
            pre_ms[k].append(pre_bwd(variants[k]))
    med = lambda d: {k: round(float(np.median(v)), 4) for k, v in d.items()}
    spread = lambda d: {k: round(float(np.max(v) - np.min(v)), 4) for k, v in d.items()}
    out = {
        "gpu": gpu, "power_limit_w": power, "config": "N=%d %dx%d SH degree 3" % (N, W, H),
        "rounds": args.rounds, "steps_per_round": args.steps,
        "step_ms": med(step_ms), "step_spread_ms": spread(step_ms),
        "preprocess_backward_ms": med(pre_ms), "preprocess_backward_spread_ms": spread(pre_ms),
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
