"""Cost of the camera models at BASELINE config 2 (1M Gaussians, SH degree 3, 1920x1080).

For pinhole, ortho, fisheye (k = 0), fisheye with COLMAP-like k1..k4, opencv (k = p = 0) and opencv with
COLMAP-like k1, k2, p1, p2: the fused training step of
GSFunctionFused (forward + backward through autograd) and the per-launch CUDA-event times
(gsb_profile_*) of the preprocess_forward, preprocess_backward, draw and draw_backward scopes, and P
(the patches the frame binned).  Each model's scene is scene.camera_model_scene: the generator's target
pixels unprojected through that model, so that P stays comparable.  The models alternate in rounds so
that clock and thermal drift hit them alike; medians over rounds are reported with the card's name and
power limit, read in the same run.  Prints one JSON line.

    python benchmarks/camera_model_step.py [--rounds 7] [--steps 10]
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

from easygaussiansplatting_b200 import _lib, ops  # noqa: E402
from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused  # noqa: E402
from easygaussiansplatting_b200.scene import (COLMAP_LIKE_FISHEYE_K, COLMAP_LIKE_OPENCV,  # noqa: E402
                                               camera_model_scene, upstream_gradient)

N, W, H, SH = 1_000_000, 1920, 1080, 48
KERNELS = ("preprocess_forward", "preprocess_backward", "draw", "draw_backward")
# label, camera_model, radial_coeffs, tangential_coeffs
MODELS = (("pinhole", "pinhole", None, None), ("ortho", "ortho", None, None), ("fisheye", "fisheye", None, None),
          ("fisheye_k", "fisheye", COLMAP_LIKE_FISHEYE_K, None), ("opencv", "opencv", None, None),
          ("opencv_k", "opencv") + COLMAP_LIKE_OPENCV)


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
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    dl = T(upstream_gradient(W, H, 0) * (3.0 * W * H))
    steps, patches = {}, {}
    for label, model, k, p in MODELS:
        sc = camera_model_scene(N, W, H, model, k, sh_dim=SH, seed=0, tangential_coeffs=p)
        cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(sc["Rcw"]), T(sc["tcw"]), T(sc["twc"]),
                     camera_model=model, radial_coeffs=k, tangential_coeffs=p)
        leaves = [T(sc[n]).requires_grad_() for n in ("pws", "shs")] + [T(sc["alphas"][:, None]).requires_grad_()] + \
                 [T(sc[n]).requires_grad_() for n in ("scales", "rots")] + \
                 [torch.zeros((N, 2), device=dev, requires_grad=True)]
        with torch.no_grad():
            pre = ops.preprocess(leaves[0], leaves[4], leaves[3], leaves[1], cam.Rcw, cam.tcw, cam.twc, cam.fx, cam.fy,
                                 cam.cx, cam.cy, W, H, camera_model=model, radial_coeffs=k, tangential_coeffs=p)
            patches[label] = int(ops.splat(H, W, pre[0], pre[1], leaves[2], pre[3], pre[2], pre[4])[4].numel())

        def fn(leaves=leaves, cam=cam):
            for p in leaves:
                p.grad = None
            image, _ = GSFunctionFused.apply(*leaves, cam)
            image.backward(dl)
        steps[label] = fn

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
        """per-launch ms of the four scopes over `steps` calls of fn"""
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

    for fn in steps.values():  # warm-up: library load, capacity bounds, allocator
        for _ in range(3):
            fn()
    gpu, power = card()
    labels = list(steps)
    res = {lb: {"step": []} for lb in labels}
    for r in range(args.rounds):
        for lb in (labels if r % 2 == 0 else labels[::-1]):
            res[lb]["step"].append(timed(steps[lb]))
            for k, v in kernels(steps[lb]).items():
                res[lb].setdefault(k, []).append(v)
    out = {
        "gpu": gpu, "power_limit_w": power, "config": "N=%d %dx%d SH degree 3" % (N, W, H),
        "rounds": args.rounds, "steps_per_round": args.steps, "fisheye_k": list(COLMAP_LIKE_FISHEYE_K),
        "opencv_k": list(COLMAP_LIKE_OPENCV[0] + COLMAP_LIKE_OPENCV[1]),
        "P": patches,
        "ms": {lb: {k: round(float(np.median(v)), 4) for k, v in d.items()} for lb, d in res.items()},
        "spread_ms": {lb: {k: round(float(np.max(v) - np.min(v)), 4) for k, v in d.items()} for lb, d in res.items()},
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
