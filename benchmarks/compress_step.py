"""Cost of the compressed export (DESIGN 3.24) on one GPU, at BASELINE config 2's size: N = 1M
Gaussians of the seeded synthetic scene, K = 65536 SH clusters, D = 45.

  kmeans_assign   ours (fused distance + argmin), CUDA events over --reps calls, and its FMA rate
                  N K D / time against the H100 SXM data sheet's 67 TFLOP/s FP32 (33.5 T FMA/s);
  torch_assign    the same assignment as chunked torch.cdist + argmin (chunks of --chunk rows),
                  alternated with ours in rounds, and how often its labels differ from ours;
  kmeans_update   one Lloyd update (the stable torch sort included);
  save / load     gau_io.save_compressed (10 iterations) and load_compressed, wall clock around a
                  device synchronise, into a temporary directory;
  distortion      the mean squared distance after each of the 10 assignments of k-means on the scene's
                  SH rows.
Prints one JSON line with the card's name and power limit read in the same run; writes nothing in
the tree.

    python benchmarks/compress_step.py [--rounds 5] [--reps 3] [--chunk 4096]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

from batch_step import card  # noqa: E402
from easygaussiansplatting_b200 import compress as cz, gau_io, ops  # noqa: E402
from easygaussiansplatting_b200.scene import synthetic_scene  # noqa: E402

DEV = "cuda"
FP32_PEAK_FMA = 67e12 / 2  # H100 SXM data sheet, dense FP32, at up to 700 W


def event_ms(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def torch_assign(x, c, chunk):
    labels = torch.empty((x.shape[0],), dtype=torch.int64, device=x.device)
    for s in range(0, x.shape[0], chunk):
        labels[s:s + chunk] = torch.cdist(x[s:s + chunk], c).argmin(dim=1)
    return labels


def wall_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--k", type=int, default=65536)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--chunk", type=int, default=4096)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "compress_step.py measures on the GPU only"
    gpu, power = card()
    N, K = a.n, a.k
    sc = synthetic_scene(N, 1920, 1080, sh_dim=48, seed=0)
    T = lambda v: torch.from_numpy(np.ascontiguousarray(v, np.float32)).to(DEV)  # noqa: E731
    al = sc["alphas"].astype(np.float64)
    params = {"pws": T(sc["pws"]), "low_shs": T(sc["shs"][:, :3]), "high_shs": T(sc["shs"][:, 3:]),
              "alphas_raw": T(np.log(al / (1 - al))[:, None]), "scales_raw": T(np.log(sc["scales"])),
              "rots_raw": T(sc["rots"])}
    x = params["high_shs"]
    D = x.shape[1]
    g = torch.Generator(device=DEV).manual_seed(0)
    c = x[torch.randperm(N, generator=g, device=DEV)[:K]].contiguous()

    ours = lambda: ops.kmeans_assign(x, c)  # noqa: E731
    theirs = lambda: torch_assign(x, c, a.chunk)  # noqa: E731
    ours(), theirs()
    t_ours, t_torch = [], []
    for _ in range(a.rounds):
        t_ours.append(event_ms(ours, a.reps))
        t_torch.append(event_ms(theirs, 1))
    labels, _ = ours()
    mismatch = int((theirs() != labels.long()).sum())
    upd = lambda: ops.kmeans_update(x, labels, c)  # noqa: E731
    upd()
    t_upd = [event_ms(upd, a.reps) for _ in range(a.rounds)]

    _, _, distortion = cz.kmeans(x, K, iters=10, generator=torch.Generator(device=DEV).manual_seed(0))
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "scene.npz")
        t_save, _ = wall_ms(lambda: gau_io.save_compressed(path, params, sh_clusters=K, iters=10,
                                                           generator=torch.Generator(device=DEV).manual_seed(0)))
        size = os.path.getsize(path)
        gau_io.load_compressed(path)
        t_load, _ = wall_ms(lambda: gau_io.load_compressed(path))

    med = float(np.median(t_ours))
    res = {"N": N, "K": K, "D": D, "gpu": gpu, "power_limit_w": power,
           "kmeans_assign_ms": round(med, 2), "kmeans_assign_ms_spread": [round(min(t_ours), 2), round(max(t_ours), 2)],
           "kmeans_assign_fma_per_s": float("%.4g" % (N * K * D / (med * 1e-3))),
           "kmeans_assign_share_of_fp32_peak": round(N * K * D / (med * 1e-3) / FP32_PEAK_FMA, 3),
           "torch_cdist_argmin_ms": round(float(np.median(t_torch)), 2),
           "torch_cdist_argmin_ms_spread": [round(min(t_torch), 2), round(max(t_torch), 2)],
           "torch_label_mismatches": mismatch,
           "kmeans_update_ms": round(float(np.median(t_upd)), 3),
           "save_compressed_ms": round(t_save, 1), "load_compressed_ms": round(t_load, 1),
           "file_bytes": size, "payload_bytes": cz.payload_bytes(N, K), "ply_bytes": 248 * N,
           "distortion": [float("%.6g" % d) for d in distortion]}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
