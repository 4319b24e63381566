"""The batch's camera gradients (DESIGN 3.22) against the batch without them and the per-view pose loop, on one
GPU and one seeded scene.

One step = forward of C views + backward of a fixed upstream gradient per view, four ways:
  batch      GSFunctionFusedBatch, poses frozen (the map gradients only);
  pose+map   GSFunctionFusedBatchPose, poses and map differentiated (the pose pass, then the batch pass);
  pose_only  GSFunctionFusedBatchPose with a frozen map (the pose pass alone: tracking C frames);
  loop       C calls of GSFunctionFusedPose, poses and map differentiated, gradients summed by autograd.
Cases: BASELINE config 5 (2M Gaussians, 8 cameras, 1920x1080) and a small-frame case (1M Gaussians, 16 cameras,
400x300).  The four alternate in rounds in one process; medians of the step time (device synchronise around each
step), then a profiled run of each for the preprocess_backward_batch scope and the other per-kernel times
(gsb_profile_*).  Prints one JSON line per case with the card's name and power limit read in the same run;
writes nothing else.

    python benchmarks/batch_pose_step.py [--rounds 5] [--steps 5] [--cases config5,small]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

from batch_step import CASES, DEV, card, kernel_times, setup, timed  # noqa: E402
from easygaussiansplatting_b200 import _lib  # noqa: E402
from easygaussiansplatting_b200.gsfunction import (GSFunctionFusedBatch, GSFunctionFusedBatchPose,  # noqa: E402
                                                   GSFunctionFusedPose)


def poses(cams, grad):
    R = torch.stack([c.Rcw for c in cams]).clone().requires_grad_(grad)
    t = torch.stack([c.tcw for c in cams]).clone().requires_grad_(grad)
    w = torch.stack([c.twc for c in cams]).clone().requires_grad_(grad)
    return R, t, w


def step_batch(cams, P, G):
    N = P["pws"].shape[0]
    us = torch.zeros((len(cams), N, 2), device=DEV, requires_grad=True)
    img, _ = GSFunctionFusedBatch.apply(P["pws"], P["shs"], P["alphas"], P["scales"], P["rots"], us, cams)
    img.backward(G)


def step_pose(cams, P, G, need_map):
    N = P["pws"].shape[0]
    us = torch.zeros((len(cams), N, 2), device=DEV, requires_grad=need_map)
    m = {k: v if need_map else v.detach() for k, v in P.items()}
    img, _ = GSFunctionFusedBatchPose.apply(m["pws"], m["shs"], m["alphas"], m["scales"], m["rots"], us,
                                            *poses(cams, True), cams)
    img.backward(G)


def step_loop(cams, P, G):
    N = P["pws"].shape[0]
    loss = 0.0
    for c, cam in enumerate(cams):
        us = torch.zeros((N, 2), device=DEV, requires_grad=True)
        R, t, w = (x[0] for x in poses([cam], True))
        img, _ = GSFunctionFusedPose.apply(P["pws"], P["shs"], P["alphas"], P["scales"], P["rots"], us, R, t, w, cam)
        loss = loss + (img * G[c]).sum()
    loss.backward()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--cases", default="config5,small")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "batch_pose_step.py measures on the GPU only"
    lib = _lib.load()
    gpu, power = card()
    for case in a.cases.split(","):
        N, C, W, H = CASES[case]
        cams, P, G = setup(N, C, W, H)
        fns = {"batch": lambda: step_batch(cams, P, G), "pose+map": lambda: step_pose(cams, P, G, True),
               "pose_only": lambda: step_pose(cams, P, G, False), "loop": lambda: step_loop(cams, P, G)}
        for f in fns.values():  # warm-up: modules, capacity bounds, allocator
            f(); f()
        for v in P.values():
            v.grad = None
        t = {k: [] for k in fns}
        for _ in range(a.rounds):
            for k, f in fns.items():
                t[k].append(timed(f, a.steps))
                for v in P.values():
                    v.grad = None
        kt = {k: kernel_times(lib, f) for k, f in fns.items()}
        res = {"case": case, "N": N, "C": C, "W": W, "H": H, "gpu": gpu, "power_limit_w": power,
               "step_ms_median": {k: round(float(np.median(v)), 3) for k, v in t.items()},
               "step_ms_spread": {k: [round(min(v), 3), round(max(v), 3)] for k, v in t.items()},
               "preprocess_backward_batch_ms": {k: v.get("preprocess_backward_batch") for k, v in kt.items()},
               "kernel_ms_per_step": kt}
        print(json.dumps(res), flush=True)
        del cams, P, G
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
