"""Cost of feature rendering at BASELINE config 2 (1M Gaussians, SH degree 3, 1920x1080).

For each feature width D: the fused training step (forward + backward through autograd, a loss on
the image and on the feature map) with GSFunctionFusedFeatures vs GSFunctionFused, the two
alternating in rounds so that clock and thermal drift hit both alike, and the CUDA-event times
(gsb_profile_*) of the feature rasterizers draw_features / draw_backward_features per step (the
sum of their ceil(D / 8) replays) next to the colour pair draw / draw_backward.  Medians over
rounds, with the card's name and power limit read in the same run.  Prints one JSON line.

    python benchmarks/features_step.py [--rounds 5] [--steps 5] [--widths 3,16,32]
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
from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused, GSFunctionFusedFeatures  # noqa: E402
from easygaussiansplatting_b200.scene import synthetic_scene, upstream_gradient  # noqa: E402

N, W, H, SH = 1_000_000, 1920, 1080, 48
KERNELS = ("draw", "draw_backward", "draw_features", "draw_backward_features")


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
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--widths", default="3,16,32")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    lib = _lib.load()
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    kid = {k: names.index(k) for k in KERNELS}
    C_d, C_ll = ctypes.c_double, ctypes.c_longlong
    sc = synthetic_scene(N, W, H, sh_dim=SH, seed=0)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(sc["Rcw"]), T(sc["tcw"]), T(sc["twc"]))
    params = {k: T(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    alphas = T(sc["alphas"][:, None]).requires_grad_()
    us0 = torch.zeros((N, 2), device=dev, requires_grad=True)
    leaves = [params["pws"], params["shs"], alphas, params["scales"], params["rots"], us0]
    dl = T(upstream_gradient(W, H, 0) * (3.0 * W * H))
    rng = np.random.default_rng(1)

    def step_rgb():
        for p in leaves:
            p.grad = None
        image, _ = GSFunctionFused.apply(params["pws"], params["shs"], alphas, params["scales"], params["rots"], us0,
                                         cam)
        image.backward(dl)

    def make_step(feat, dF):
        def step():
            for p in leaves + [feat]:
                p.grad = None
            image, fmap, _ = GSFunctionFusedFeatures.apply(params["pws"], params["shs"], alphas, params["scales"],
                                                           params["rots"], us0, feat, cam)
            torch.autograd.backward([image, fmap], [dl, dF])
        return step

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
        """ms per step of each rasterizer kernel (all its launches) over `steps` calls of fn"""
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

    gpu, power = card()
    results = {}
    for D in (int(x) for x in args.widths.split(",")):
        feat = T(rng.normal(size=(N, D)).astype(np.float32)).requires_grad_()
        dF = T(rng.normal(size=(D, H, W)).astype(np.float32) / np.float32(D * H * W))
        step_feat = make_step(feat, dF)
        for fn in (step_rgb, step_feat):  # warm-up: library load, capacity bounds, allocator
            for _ in range(3):
                fn()
        res = {"step_rgb": [], "step_features": []}
        res.update({k: [] for k in KERNELS})
        for r in range(args.rounds):
            order = (step_rgb, step_feat) if r % 2 == 0 else (step_feat, step_rgb)
            for fn in order:
                res["step_rgb" if fn is step_rgb else "step_features"].append(timed(fn))
                for k, v in kernels(fn).items():
                    if fn is step_feat or not k.endswith("features"):
                        res[k].append(v)
        med = {k: float(np.median(v)) for k, v in res.items() if v}
        results["D=%d" % D] = {
            "ms": {k: round(v, 4) for k, v in med.items()},
            "spread_ms": {k: round(float(np.max(v) - np.min(v)), 4) for k, v in res.items() if v},
            "replays": (D + 7) // 8,
            "features_vs_colour": {
                "forward_kernel": round(med["draw_features"] / med["draw"], 4),
                "backward_kernel": round(med["draw_backward_features"] / med["draw_backward"], 4),
                "step_overhead": round(med["step_features"] / med["step_rgb"] - 1.0, 4),
            },
        }
        del feat, dF, step_feat
    out = {"gpu": gpu, "power_limit_w": power, "config": "N=%d %dx%d SH degree 3" % (N, W, H),
           "rounds": args.rounds, "steps_per_round": args.steps, "widths": results}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
