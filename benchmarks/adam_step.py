"""Cost of one Adam step over the reference's six Gaussian tensors at N = 1M (59 floats per
Gaussian; DESIGN 3.12).

Rows, all on the same params, grads and state layout:
  ours_dense               GaussianAdam.step()
  ours_selective_<f>       GaussianAdam.step(visibility=mask), a random mask of visible fraction f
  ours_selective_frame     the same with the fused frame's own mask (depths > 0.2) on the bench scene
                           (1M synthetic Gaussians, 1920x1080, SH degree 3)
  torch_foreach            torch.optim.Adam default (foreach for CUDA params)
  torch_fused              torch.optim.Adam(fused=True)
  torch_selective          selective Adam composed from torch ops (gather the visible rows, the
                           foreach update on them, scatter back)
Each row is CUDA events around one step() call (host work included), replayed in rounds that
alternate the rows so that clock drift hits all alike; medians over the rounds after a warm-up.
For our rows the kernel's own time comes from the library's per-kernel events.  Achieved GB/s =
the algorithmic bytes (28 B per updated element: read p, g, m, v, write p, m, v; plus N bytes of
mask for the selective rows) over the time.  The card's name and power limit are read in the same
run.  Prints one JSON line.

    python benchmarks/adam_step.py [--rounds 30] [--n 1000000]
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
from easygaussiansplatting_b200.gau_io import adam_groups  # noqa: E402
from easygaussiansplatting_b200.optim import GaussianAdam  # noqa: E402

WIDTHS = dict(pws=3, low_shs=3, high_shs=45, alphas_raw=1, scales_raw=3, rots_raw=4)
FLOATS = sum(WIDTHS.values())  # 59


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(q.splitlines()[0])
    except Exception:
        power = None
    return name, power


def frame_mask(N, dev):
    """the visibility mask GSFunctionFused returns for the bench scene's camera"""
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused
    from easygaussiansplatting_b200.scene import synthetic_scene
    W, H = 1920, 1080
    sc = synthetic_scene(N, W, H, sh_dim=48, seed=0)
    T = lambda a: torch.from_numpy(a).to(dev)  # noqa: E731
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(sc["Rcw"]), T(sc["tcw"]), T(sc["twc"]))
    with torch.no_grad():
        _, mask = GSFunctionFused.apply(T(sc["pws"]), T(sc["shs"]), T(sc["alphas"][:, None]), T(sc["scales"]),
                                        T(sc["rots"]), torch.zeros((N, 2), device=dev), cam)
    return mask


def torch_selective_step(P, G, M, V, vis, t, lrs, b1=0.9, b2=0.999, eps=1e-15):
    """selective Adam from torch ops: the visible rows gathered, torch's foreach update, scattered back"""
    idx = vis.nonzero()[:, 0]
    bc1, bc2 = 1 - b1 ** t, (1 - b2 ** t) ** 0.5
    for k in P:
        g = G[k].index_select(0, idx)
        m = M[k].index_select(0, idx).lerp_(g, 1 - b1)
        v = V[k].index_select(0, idx).mul_(b2).addcmul_(g, g, value=1 - b2)
        denom = v.sqrt().div_(bc2).add_(eps)
        P[k].index_copy_(0, idx, P[k].index_select(0, idx).addcdiv_(m, denom, value=-lrs[k] / bc1))
        M[k].index_copy_(0, idx, m)
        V[k].index_copy_(0, idx, v)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--n", type=int, default=1_000_000)
    args = ap.parse_args()
    N = args.n
    dev = torch.device("cuda", 0)
    lib = _lib.load()
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    kid = names.index("adam")
    gen = torch.Generator(device=dev).manual_seed(0)
    base = {k: torch.randn((N, w), device=dev, generator=gen) for k, w in WIDTHS.items()}
    grads = {k: torch.randn((N, w), device=dev, generator=gen) * 1e-3 for k, w in WIDTHS.items()}

    def setup(make):
        params = {k: torch.nn.Parameter(v.clone()) for k, v in base.items()}
        for k, p in params.items():
            p.grad = grads[k].clone()
        opt = make(adam_groups(params))
        opt.step()  # creates the state
        return params, opt

    masks = {f: torch.rand(N, device=dev, generator=gen) < f for f in (0.5, 0.2)}
    masks[1.0] = torch.ones(N, dtype=torch.bool, device=dev)
    masks["frame"] = frame_mask(N, dev)
    ours = setup(lambda g: GaussianAdam(g, eps=1e-15))
    foreach = setup(lambda g: torch.optim.Adam(g, eps=1e-15))
    fused = setup(lambda g: torch.optim.Adam(g, eps=1e-15, fused=True))
    lrs = {g["name"]: g["lr"] for g in ours[1].param_groups}
    TP = {k: v.clone() for k, v in base.items()}
    TM = {k: torch.zeros_like(v) for k, v in base.items()}
    TV = {k: torch.zeros_like(v) for k, v in base.items()}
    tstep = [0]

    def torch_sel(mask):
        tstep[0] += 1
        torch_selective_step(TP, grads, TM, TV, mask, tstep[0], lrs)

    rows = {"ours_dense": (lambda: ours[1].step(), None)}
    for f in (1.0, 0.5, 0.2, "frame"):
        rows["ours_selective_%s" % f] = ((lambda m: lambda: ours[1].step(visibility=m))(masks[f]), masks[f])
    rows["torch_foreach"] = (lambda: foreach[1].step(), None)
    rows["torch_fused"] = (lambda: fused[1].step(), None)
    rows["torch_selective_0.5"] = ((lambda m: lambda: torch_sel(m))(masks[0.5]), masks[0.5])
    rows["torch_selective_frame"] = ((lambda m: lambda: torch_sel(m))(masks["frame"]), masks["frame"])

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    def kernel_ms(fn):
        C_d, C_ll = ctypes.c_double, ctypes.c_longlong
        lib.gsb_profile_enable(1)
        lib.gsb_profile_read(kid, ctypes.byref(C_d()), ctypes.byref(C_ll()))
        fn()
        torch.cuda.synchronize()
        lib.gsb_profile_enable(0)
        ms, cnt = C_d(), C_ll()
        lib.gsb_profile_read(kid, ctypes.byref(ms), ctypes.byref(cnt))
        return ms.value

    for fn, _ in rows.values():  # warm-up
        for _ in range(3):
            timed(fn)
    res = {k: [] for k in rows}
    kres = {k: [] for k in rows if k.startswith("ours")}
    order = list(rows)
    for r in range(args.rounds):
        for k in (order if r % 2 == 0 else order[::-1]):
            res[k].append(timed(rows[k][0]))
            if k in kres:
                kres[k].append(kernel_ms(rows[k][0]))
    gpu, power = card()
    out = {"gpu": gpu, "power_limit_w": power, "N": N, "floats_per_gaussian": FLOATS, "rounds": args.rounds,
           "frame_visible_fraction": round(float(masks["frame"].float().mean()), 4), "rows": {}}
    for k, (_, mask) in rows.items():
        upd = N * FLOATS if mask is None else int(mask.sum()) * FLOATS
        nbytes = 28 * upd + (N if mask is not None else 0)
        ms = float(np.median(res[k]))
        row = {"ms": round(ms, 4), "spread_ms": round(float(np.max(res[k]) - np.min(res[k])), 4),
               "algorithmic_bytes": nbytes, "gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1),
               "datasheet_bound_ms": round(nbytes / 3.35e12 * 1e3, 4)}
        if k in kres:
            kms = float(np.median(kres[k]))
            row["kernel_ms"] = round(kms, 4)
            row["kernel_gb_per_s"] = round(nbytes / (kms * 1e-3) / 1e9, 1)
        out["rows"][k] = row
    print(json.dumps(out))


if __name__ == "__main__":
    main()
