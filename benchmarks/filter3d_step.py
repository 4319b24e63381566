"""Cost of the Mip-Splatting 3D smoothing filter.

1. ops.filter3d at N = 1M Gaussians and C in {50, 300, 1000} training cameras, against a torch
   implementation of the same definition (a loop over the cameras, as Mip-Splatting's
   compute_3D_filter runs it) on the same GPU; both must give the same filter.
2. The fused training step at BASELINE config 2 (1M Gaussians, SH degree 3, 1920x1080) with the
   filter off and on, each with antialiasing off and on, alternating in rounds (rotated order), with
   the per-launch CUDA-event time of the `filter3d_apply` and `filter3d_backward` profile scopes.
Medians over rounds, with the card's name and power limit read in the same run.  Prints one JSON line.

    python benchmarks/filter3d_step.py [--rounds 5] [--steps 10]
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

from antialias_step import card  # noqa: E402
from easygaussiansplatting_b200 import _lib, ops  # noqa: E402
from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused  # noqa: E402
from easygaussiansplatting_b200.scene import synthetic_scene, upstream_gradient  # noqa: E402

N, W, H, SH = 1_000_000, 1920, 1080, 48


def torch_filter3d(pws, table, variance=0.2):
    """the same definition in torch, one camera at a time (fp32, the kernels' operation order)"""
    best = torch.full((pws.shape[0],), float("inf"), device=pws.device)
    for row in table:
        R, t = row[:9].view(3, 3), row[9:12]
        fx, fy, cx, cy, w, h = row[12:18]
        z = torch.addcmul(torch.addcmul(torch.addcmul(t[2], R[2, 2], pws[:, 2]), R[2, 1], pws[:, 1]), R[2, 0], pws[:, 0])
        x = torch.addcmul(torch.addcmul(torch.addcmul(t[0], R[0, 2], pws[:, 2]), R[0, 1], pws[:, 1]), R[0, 0], pws[:, 0])
        y = torch.addcmul(torch.addcmul(torch.addcmul(t[1], R[1, 2], pws[:, 2]), R[1, 1], pws[:, 1]), R[1, 0], pws[:, 0])
        keep = z >= 0.2
        zi = 1.0 / torch.where(keep, z, torch.ones_like(z))
        ux, uy = x * fx * zi + cx, y * fy * zi + cy
        lo, hi = torch.tensor(-0.15, device=pws.device), torch.tensor(1.15, device=pws.device)
        seen = keep & (ux >= lo * w) & (ux <= hi * w) & (uy >= lo * h) & (uy <= hi * h)
        best = torch.where(seen, torch.minimum(best, z), best)
    seen = torch.isfinite(best)
    if not seen.any():
        return torch.zeros_like(best)
    d = torch.where(seen, best, best[seen].max())
    return (variance ** 0.5) * d / table[:, 12].max()


def ring(C, dev, seed=0):
    rng = np.random.default_rng(seed)
    rows = np.zeros((C, 20), np.float32)
    for k in range(C):
        a = 2 * np.pi * k / C
        eye = np.array([8 * np.cos(a), rng.uniform(-1, 1), 8 * np.sin(a) + 7.0])
        z = np.array([0.0, 0.0, 7.0]) - eye
        z /= np.linalg.norm(z)
        x = np.cross(z, [0.0, 1.0, 0.0]); x /= np.linalg.norm(x)
        R = np.stack([x, np.cross(z, x), z])
        rows[k, :9], rows[k, 9:12] = R.reshape(-1), -R @ eye
        rows[k, 12:18] = [1663.0 * rng.uniform(0.9, 1.1), 1663.0, W / 2, H / 2, W, H]
    return torch.from_numpy(rows).to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    lib = _lib.load()
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    sc = synthetic_scene(N, W, H, sh_dim=SH, seed=0)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    pws = T(sc["pws"])

    def timed(fn, steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    gpu, power = card()
    filt = {}
    for C in (50, 300, 1000):
        table = ring(C, dev, seed=C)
        a, b = ops.filter3d(pws, table), torch_filter3d(pws, table)
        # the torch loop rounds like the kernel up to FMA contraction, which can flip a visibility
        # decision that lies on a bound: count the rows that differ rather than ask for bits
        diff = int(((a - b).abs() > 1e-6 * b.abs()).sum())
        assert diff <= max(1, N // 100000), (C, diff)
        kern = [timed(lambda: ops.filter3d(pws, table), 5) for _ in range(args.rounds)]
        loop = [timed(lambda: torch_filter3d(pws, table), 1) for _ in range(max(2, args.rounds // 2))]
        filt[C] = {"kernel_ms": round(float(np.median(kern)), 4), "torch_loop_ms": round(float(np.median(loop)), 3),
                   "rows_differing": diff, "seen_fraction": round(float((a < a.max()).float().mean()), 4)}
    # ---- the fused step with the filter off / on, AA off / on
    cams = {aa: Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(sc["Rcw"]), T(sc["tcw"]), T(sc["twc"]),
                       antialiased=aa) for aa in (False, True)}
    f3 = ops.filter3d(pws, ops.camera_table([cams[False]]))
    params = {k: T(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    alphas = T(sc["alphas"][:, None]).requires_grad_()
    us0 = torch.zeros((N, 2), device=dev, requires_grad=True)
    leaves = [params["pws"], params["shs"], alphas, params["scales"], params["rots"], us0]
    dl = T(upstream_gradient(W, H, 0) * (3.0 * W * H))

    def step(aa, filtered):
        for p in leaves:
            p.grad = None
        with torch.profiler.record_function("filter3d_step"):
            out = GSFunctionFused.apply(*leaves, cams[aa], *((f3,) if filtered else ()))
            out[0].backward(dl)

    variants = {("aa_" if aa else "plain_") + ("filter" if f else "nofilter"): (lambda aa=aa, f=f: step(aa, f))
                for aa in (False, True) for f in (False, True)}
    scopes = ("filter3d_apply", "filter3d_backward", "preprocess_forward", "preprocess_backward")
    C_d, C_ll = ctypes.c_double, ctypes.c_longlong

    def profiled(fn):
        lib.gsb_profile_enable(1)
        for s in scopes:
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

    for fn in variants.values():
        for _ in range(3):
            fn()
    keys = list(variants)
    step_ms = {k: [] for k in keys}
    scope_ms = {k: {} for k in keys}
    for r in range(args.rounds):
        for k in keys[r % len(keys):] + keys[:r % len(keys)]:
            step_ms[k].append(timed(variants[k], args.steps))
            for s, v in profiled(variants[k]).items():
                scope_ms[k].setdefault(s, []).append(v)
    med = lambda v: round(float(np.median(v)), 4)
    print(json.dumps({
        "gpu": gpu, "power_limit_w": power, "config": "N=%d %dx%d SH degree 3" % (N, W, H), "rounds": args.rounds,
        "filter3d": filt, "step_ms": {k: med(v) for k, v in step_ms.items()},
        "step_spread_ms": {k: round(float(np.max(v) - np.min(v)), 4) for k, v in step_ms.items()},
        "scope_ms": {k: {s: med(v) for s, v in d.items()} for k, d in scope_ms.items()},
    }))


if __name__ == "__main__":
    main()
