"""Cost of the intrinsics gradient (DESIGN 3.23) on one GPU and one seeded scene.

One step = forward + backward of a fixed upstream gradient, four ways:
  none        the map gradients only (poses and intrinsics fixed);
  pose        poses and map differentiated (the pose pass, then the map pass);
  pose+intr   poses, intrinsics and map differentiated (the pose + intrinsics pass, then the map pass);
  intr_only   the intrinsics alone, a frozen map and fixed poses (the pose + intrinsics pass alone).
Cases: BASELINE config 2 with one camera (1M Gaussians, 1920x1080, GSFunctionFusedPose) and config 5
(2M Gaussians, 8 cameras, 1920x1080, GSFunctionFusedBatchPose).  The intrinsics travel as a CPU tensor.
The arms alternate in rounds in one process; medians of the step time (device synchronise around each
step), then a profiled run of each for the camera pass's scope (preprocess_backward[_batch]).  Prints one
JSON line per case with the card's name and power limit read in the same run; writes nothing else.

    python benchmarks/calib_step.py [--rounds 5] [--steps 5] [--cases config2,config5]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

from batch_step import DEV, card, kernel_times, setup, timed  # noqa: E402
from easygaussiansplatting_b200 import _lib  # noqa: E402
from easygaussiansplatting_b200.gsfunction import GSFunctionFusedBatchPose, GSFunctionFusedPose  # noqa: E402

CASES = {"config2": (1_000_000, 1, 1920, 1080), "config5": (2_000_000, 8, 1920, 1080)}
ARMS = {"none": (True, False, False), "pose": (True, True, False), "pose+intr": (True, True, True),
        "intr_only": (False, False, True)}


def step(cams, P, G, need_map, need_pose, need_intr):
    C, N = len(cams), P["pws"].shape[0]
    m = {k: v if need_map else v.detach() for k, v in P.items()}
    R = torch.stack([c.Rcw for c in cams]).clone().requires_grad_(need_pose)
    t = torch.stack([c.tcw for c in cams]).clone().requires_grad_(need_pose)
    w = torch.stack([c.twc for c in cams]).clone().requires_grad_(need_pose)
    intr = torch.tensor([[c.fx, c.fy, c.cx, c.cy, 0.0, 0.0, 0.0, 0.0] for c in cams], requires_grad=need_intr)
    if C == 1:
        us = torch.zeros((N, 2), device=DEV, requires_grad=need_map)
        img, _ = GSFunctionFusedPose.apply(m["pws"], m["shs"], m["alphas"], m["scales"], m["rots"], us, R[0], t[0],
                                           w[0], cams[0], None, None, intr[0])
        img.backward(G[0])
    else:
        us = torch.zeros((C, N, 2), device=DEV, requires_grad=need_map)
        img, _ = GSFunctionFusedBatchPose.apply(m["pws"], m["shs"], m["alphas"], m["scales"], m["rots"], us, R, t, w,
                                                cams, None, intr)
        img.backward(G)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--cases", default="config2,config5")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "calib_step.py measures on the GPU only"
    lib = _lib.load()
    gpu, power = card()
    for case in a.cases.split(","):
        N, C, W, H = CASES[case]
        cams, P, G = setup(N, C, W, H)
        fns = {k: (lambda f=f: step(cams, P, G, *f)) for k, f in ARMS.items()}
        for f in fns.values():  # warm-up: modules, capacity bounds, allocator
            f(); f()
        t = {k: [] for k in fns}
        for _ in range(a.rounds):
            for k, f in fns.items():
                t[k].append(timed(f, a.steps))
                for v in P.values():
                    v.grad = None
        scope = "preprocess_backward" if C == 1 else "preprocess_backward_batch"
        kt = {k: kernel_times(lib, f) for k, f in fns.items()}
        res = {"case": case, "N": N, "C": C, "W": W, "H": H, "gpu": gpu, "power_limit_w": power,
               "step_ms_median": {k: round(float(np.median(v)), 3) for k, v in t.items()},
               "step_ms_spread": {k: [round(min(v), 3), round(max(v), 3)] for k, v in t.items()},
               scope + "_ms": {k: v.get(scope) for k, v in kt.items()}}
        print(json.dumps(res), flush=True)
        del cams, P, G
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
