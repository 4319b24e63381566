"""Cost of the bilateral-grid colour correction (DESIGN 3.20) at 1920x1080 with M = 300 grids of
16 x 16 x 8.

- The kernels: CUDA-event times (gsb_profile_*) of bilagrid_slice, bilagrid_slice_backward and
  bilagrid_tv, with their algorithmic bytes from the shapes and the share of the 3.35 TB/s
  data-sheet HBM3 bound those bytes give.  Forward: read rgb, write out (6 planes); backward: read
  rgb and dL/dout, write dL/drgb (9 planes); TV: read and write the grids once.  The grid window
  and the per-CTA gradient adds are not counted.
- The ops against the torch composition on the same inputs: F.grid_sample over the 5D grid and
  its autograd backward (oracle/bilagrid_oracle.py torch_slice), and the TV in torch.  Both sides
  include allocating and zeroing the dense [M, 12, L, Y, X] grid gradient.
- The fused training step at BASELINE config 2 (1M Gaussians, SH degree 3, 1920x1080; forward,
  gau_loss, backward, no optimiser step) with and without the grid and its TV.
Each pair alternates in rounds in the same process; medians, with the card's name and power limit
read in the same run.  Prints one JSON line.

    python benchmarks/bilagrid_step.py [--rounds 7] [--steps 20]
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
from easygaussiansplatting_b200.bilagrid import BilateralGrid, bilateral_slice, total_variation  # noqa: E402
from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused  # noqa: E402
from easygaussiansplatting_b200.loss import gau_loss  # noqa: E402
from easygaussiansplatting_b200.scene import synthetic_scene  # noqa: E402
from oracle.bilagrid_oracle import torch_slice  # noqa: E402

W, H, M, L, GY, GX = 1920, 1080, 300, 8, 16, 16
N, SH = 1_000_000, 48
HBM_BPS = 3.35e12  # NVIDIA H100 SXM data sheet
KERNELS = ("bilagrid_slice", "bilagrid_slice_backward", "bilagrid_tv")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(q.splitlines()[0])
    except Exception:
        power = None
    return name, power


def algorithmic_bytes():
    plane = 4 * W * H
    grids = 4 * M * 12 * L * GY * GX
    return {"bilagrid_slice": 6 * plane, "bilagrid_slice_backward": 9 * plane, "bilagrid_tv": 2 * grids}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    lib = _lib.load()
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    kid = {k: names.index(k) for k in KERNELS}
    C_d, C_ll = ctypes.c_double, ctypes.c_longlong
    rng = np.random.default_rng(0)
    bil = BilateralGrid(M, grid_X=GX, grid_Y=GY, grid_L=L, device=dev)
    with torch.no_grad():
        bil.grids.add_(torch.from_numpy((0.05 * rng.standard_normal(bil.grids.shape)).astype(np.float32)).to(dev))
    grids = bil.grids.detach()
    rgb = torch.from_numpy(rng.uniform(0, 1, (3, H, W)).astype(np.float32)).to(dev)
    dout = torch.from_numpy(rng.standard_normal((3, H, W)).astype(np.float32)).to(dev)
    dgrids = torch.zeros_like(grids)
    i = 137

    def timed(fn, steps=None):
        steps = steps or args.steps
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    def kernel_ms(fn, name):
        lib.gsb_profile_enable(1)
        for k in kid.values():  # drop what earlier calls recorded
            lib.gsb_profile_read(k, ctypes.byref(C_d()), ctypes.byref(C_ll()))
        for _ in range(args.steps):
            fn()
        torch.cuda.synchronize()
        lib.gsb_profile_enable(0)
        ms, cnt = C_d(), C_ll()
        lib.gsb_profile_read(kid[name], ctypes.byref(ms), ctypes.byref(cnt))
        return ms.value / max(cnt.value, 1)

    k_fwd = lambda: ops.bilagrid_slice(grids, rgb, i)  # noqa: E731
    k_bwd = lambda: ops.bilagrid_sliceB(grids, rgb, i, dout, dloss_dgrids=dgrids)  # noqa: E731
    k_tv = lambda: ops.bilagrid_tv(grids)  # noqa: E731

    def ours_fwd_bwd():
        g = grids.clone().requires_grad_()
        r = rgb.clone().requires_grad_()
        bilateral_slice(g, r, i).backward(dout)

    def torch_fwd():
        with torch.no_grad():
            torch_slice(grids, rgb, i)

    def torch_fwd_bwd():
        g = grids.clone().requires_grad_()
        r = rgb.clone().requires_grad_()
        torch_slice(g, r, i).backward(dout)

    def torch_tv():
        g = grids.clone().requires_grad_()
        sum((g.diff(dim=a) ** 2).mean() for a in (2, 3, 4)).backward()

    def ours_tv():
        g = grids.clone().requires_grad_()
        total_variation(g).backward()

    # the two slices agree before anything is timed
    with torch.no_grad():
        agree = float((ops.bilagrid_slice(grids, rgb, i) - torch_slice(grids, rgb, i)).abs().max())

    gpu, power = card()
    pairs = {"slice": (k_fwd, torch_fwd), "slice_fwd_bwd": (ours_fwd_bwd, torch_fwd_bwd), "tv_fwd_bwd": (ours_tv, torch_tv)}
    for a, b in pairs.values():  # warm-up
        for _ in range(3):
            a(), b()
    res = {}
    for r in range(args.rounds):
        for key, (a, b) in pairs.items():
            order = ((a, "ours"), (b, "torch")) if r % 2 == 0 else ((b, "torch"), (a, "ours"))
            for fn, side in order:
                res.setdefault("%s_%s_ms" % (key, side), []).append(timed(fn))
        res.setdefault("bilagrid_slice_kernel_ms", []).append(kernel_ms(k_fwd, "bilagrid_slice"))
        res.setdefault("bilagrid_slice_backward_kernel_ms", []).append(kernel_ms(k_bwd, "bilagrid_slice_backward"))
        res.setdefault("bilagrid_tv_kernel_ms", []).append(kernel_ms(k_tv, "bilagrid_tv"))
    del dgrids
    torch.cuda.empty_cache()

    # the fused config-2 step with and without the grid
    sc = synthetic_scene(N, W, H, sh_dim=SH, seed=0)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(sc["Rcw"]), T(sc["tcw"]), T(sc["twc"]))
    P = [T(sc[k]).requires_grad_() for k in ("pws", "shs")]
    alphas = T(sc["alphas"][:, None]).requires_grad_()
    sr = [T(sc[k]).requires_grad_() for k in ("scales", "rots")]
    us = torch.zeros((N, 2), device=dev, requires_grad=True)
    gt = rgb

    def step(with_grid):
        image, _ = GSFunctionFused.apply(P[0], P[1], alphas, sr[0], sr[1], us, cam)
        if with_grid:
            loss = gau_loss(bil(image, i), gt) + 10.0 * bil.tv_loss()
        else:
            loss = gau_loss(image, gt)
        loss.backward()
        for t in (*P, alphas, *sr, us, bil.grids):
            t.grad = None

    plain, graded = (lambda: step(False)), (lambda: step(True))
    for _ in range(3):
        plain(), graded()
    for r in range(args.rounds):
        order = ((plain, "plain"), (graded, "grid")) if r % 2 == 0 else ((graded, "grid"), (plain, "plain"))
        for fn, side in order:
            res.setdefault("config2_step_%s_ms" % side, []).append(timed(fn, steps=max(3, args.steps // 4)))

    med = {k: float(np.median(v)) for k, v in res.items()}
    nbytes = algorithmic_bytes()
    out = {"gpu": gpu, "power_limit_w": power,
           "config": "%dx%d, M=%d grids of X=%d Y=%d L=%d; step: N=%d SH degree 3" % (W, H, M, GX, GY, L, N),
           "rounds": args.rounds, "steps_per_round": args.steps,
           "ms": {k: round(v, 4) for k, v in med.items()},
           "spread_ms": {k: round(float(np.max(v) - np.min(v)), 4) for k, v in res.items()},
           "algorithmic_mb": {k: round(v / 1e6, 2) for k, v in nbytes.items()},
           "hbm_floor_us": {k: round(v / HBM_BPS * 1e6, 2) for k, v in nbytes.items()},
           "share_of_hbm_bound": {k: round(nbytes[k] / HBM_BPS * 1e3 / med[k + "_kernel_ms"], 3) for k in KERNELS},
           "slice_vs_torch": round(med["slice_ours_ms"] / med["slice_torch_ms"], 4),
           "slice_fwd_bwd_vs_torch": round(med["slice_fwd_bwd_ours_ms"] / med["slice_fwd_bwd_torch_ms"], 4),
           "tv_fwd_bwd_vs_torch": round(med["tv_fwd_bwd_ours_ms"] / med["tv_fwd_bwd_torch_ms"], 4),
           "config2_step_grid_vs_plain": round(med["config2_step_grid_ms"] / med["config2_step_plain_ms"], 4),
           "slice_vs_grid_sample_max_abs_diff": agree}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
