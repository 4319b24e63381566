"""Cost of antialiasing at BASELINE config 2 (1M Gaussians, SH degree 3, 1920x1080).

The fused training step (forward + backward through autograd) with cam.antialiased off and on, each
as RGB (GSFunctionFused) and RGB-D (GSFunctionFusedRGBD).  Besides the step time, the per-launch
CUDA-event time of the `preprocess_forward`, `preprocess_backward`, `draw[_rgbd]` and
`draw_backward[_rgbd]` profile scopes: antialiasing adds a little per-Gaussian work, and alpha_eff
<= alpha shrinks every record's culling footprint, which the rasterizers may feel.  The four
variants alternate in rounds (rotated order) so that clock and thermal drift hit all alike; medians
over rounds are reported with the card's name and power limit, read in the same run.  Prints one
JSON line.

    python benchmarks/antialias_step.py [--rounds 7] [--steps 10]
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
    scopes = ("preprocess_forward", "preprocess_backward", "draw", "draw_backward", "draw_rgbd", "draw_backward_rgbd")
    sc = synthetic_scene(N, W, H, sh_dim=SH, seed=0)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    cams = {aa: Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(sc["Rcw"]), T(sc["tcw"]), T(sc["twc"]),
                       antialiased=aa) for aa in (False, True)}
    params = {k: T(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    alphas = T(sc["alphas"][:, None]).requires_grad_()
    us0 = torch.zeros((N, 2), device=dev, requires_grad=True)
    leaves = [params["pws"], params["shs"], alphas, params["scales"], params["rots"], us0]
    dl = T(upstream_gradient(W, H, 0) * (3.0 * W * H))
    rng = np.random.default_rng(1)
    dld, dla = T(rng.normal(size=(H, W)).astype(np.float32) / 12.0), T(rng.normal(size=(H, W)).astype(np.float32))

    def step(rgbd, aa):
        for p in leaves:
            p.grad = None
        out = (GSFunctionFusedRGBD if rgbd else GSFunctionFused).apply(*leaves, cams[aa])
        if rgbd:
            torch.autograd.backward(list(out[:3]), [dl, dld, dla])
        else:
            out[0].backward(dl)

    variants = {("rgbd_" if r else "rgb_") + ("aa" if aa else "plain"): (lambda r=r, aa=aa: step(r, aa))
                for r in (False, True) for aa in (False, True)}

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

    def profiled(fn):
        """per-launch ms of each scope over `steps` calls of fn (scopes that did not run: absent)"""
        lib.gsb_profile_enable(1)
        for s in scopes:  # drop earlier records
            lib.gsb_profile_read(names.index(s), ctypes.byref(C_d()), ctypes.byref(C_ll()))
        for _ in range(args.steps):
            fn()
        torch.cuda.synchronize()
        lib.gsb_profile_enable(0)
        out = {}
        for s in scopes:
            ms, cnt = C_d(), C_ll()
            lib.gsb_profile_read(names.index(s), ctypes.byref(ms), ctypes.byref(cnt))
            if cnt.value:
                out[s] = ms.value / cnt.value
        return out

    for fn in variants.values():  # warm-up: library load, capacity bounds, allocator
        for _ in range(3):
            fn()
    gpu, power = card()
    keys = list(variants)
    step_ms = {k: [] for k in keys}
    scope_ms = {k: {} for k in keys}
    for r in range(args.rounds):
        for k in keys[r % len(keys):] + keys[:r % len(keys)]:
            step_ms[k].append(timed(variants[k]))
            for s, v in profiled(variants[k]).items():
                scope_ms[k].setdefault(s, []).append(v)
    med = lambda v: round(float(np.median(v)), 4)
    out = {
        "gpu": gpu, "power_limit_w": power, "config": "N=%d %dx%d SH degree 3" % (N, W, H),
        "rounds": args.rounds, "steps_per_round": args.steps,
        "step_ms": {k: med(v) for k, v in step_ms.items()},
        "step_spread_ms": {k: round(float(np.max(v) - np.min(v)), 4) for k, v in step_ms.items()},
        "scope_ms": {k: {s: med(v) for s, v in d.items()} for k, d in scope_ms.items()},
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
