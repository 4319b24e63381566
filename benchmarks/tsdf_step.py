"""Cost of mesh extraction (DESIGN 3.17) at the size 2D Gaussian Splatting meshes at: 64 views of
1920x1080 depth and colour fused into a 512^3 coloured grid, then marching cubes.

The depth maps are median depths (where alpha >= 0.5) and the colour the image that
GSFunctionSurfelGeometry renders of the synthetic scene (1M surfels) from 64 cameras on a ring
around it.  Timed with CUDA events, the variants taking turns over rounds: integration one view
per launch (64 launches), integration 16 views per launch (4 launches), and extraction (plan, host
read of the counts, emit).  Reported: median ms, and the algorithmic bytes over kernel time against
the H100 SXM data sheet's 3.35 TB/s -- the grid's state read and written once per launch (tsdf,
weight, colour: 40 B per point) plus every depth and colour pixel read once -- with the card's
name and power limit read in the same run.  Also checks that the two integrations give
bit-identical grids.  Prints one JSON line.

    python benchmarks/tsdf_step.py [--rounds 5]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from easygaussiansplatting_b200 import ops  # noqa: E402
from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionSurfelGeometry  # noqa: E402
from easygaussiansplatting_b200.mesh import TSDFVolume  # noqa: E402
from easygaussiansplatting_b200.scene import synthetic_scene  # noqa: E402

N_SURFELS, W, H, V, NGRID, BATCH = 1_000_000, 1920, 1080, 64, 512, 16
PEAK_BPS = 3.35e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(q.splitlines()[0])
    except Exception:
        power = None
    return name, power


def ring_cameras(sc, dev, center, radius):
    """V cameras on a horizontal ring around center, 15 degrees above it, looking at it"""
    cams = []
    for k in range(V):
        a = 2 * math.pi * k / V
        c = center + radius * np.array([math.sin(a), -math.sin(math.radians(15)), -math.cos(a)])
        z = (center - c) / np.linalg.norm(center - c)
        x = np.cross([0.0, -1.0, 0.0], z)
        x /= np.linalg.norm(x)
        R = np.stack([x, np.cross(z, x), z])
        T = lambda a_: torch.tensor(a_, dtype=torch.float32, device=dev)  # noqa: E731
        cams.append(Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(R), T(-R @ c)))
    return cams


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    sc = synthetic_scene(N_SURFELS, W, H, sh_dim=48, seed=0)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    P = [T(sc[k]) for k in ("pws", "shs")]
    alphas, scales, rots = T(sc["alphas"][:, None]), T(sc["scales"]), T(sc["rots"])
    us = torch.zeros((N_SURFELS, 2), device=dev)
    center = np.array([0.0, 0.0, 7.0])
    cams = ring_cameras(sc, dev, center, 9.0)
    depth = torch.empty((V, H, W), device=dev)
    color = torch.empty((V, 3, H, W), device=dev)
    with torch.no_grad():
        for k, cam in enumerate(cams):
            image, _, alpha, _, _, median, _ = GSFunctionSurfelGeometry.apply(P[0], P[1], alphas, scales, rots, us,
                                                                              cam)
            depth[k] = torch.where(alpha >= 0.5, median, torch.zeros_like(median))
            color[k] = image.clamp(0, 1)
    lo, hi = center - 6.0, center + 6.0
    vol = TSDFVolume(lo, hi, 12.0 / (NGRID - 1), device=dev)
    assert vol.dims == (NGRID,) * 3
    table = ops.camera_table(cams, device=dev)
    Ng = NGRID ** 3

    def reset():
        vol.tsdf.fill_(1.0), vol.weight.zero_(), vol.color.zero_()

    def integrate(batch):
        for v0 in range(0, V, batch):
            ops.tsdf_integrate(vol.tsdf, vol.weight, vol.color, vol.origin, vol.voxel_size, vol.trunc,
                               vol.depth_trunc, table[v0:v0 + batch], depth[v0:v0 + batch], color[v0:v0 + batch])

    def timed(fn):
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b), out

    # warm-up of every variant, and the bit-identity check at full size
    reset(); integrate(1); one = [t.clone() for t in (vol.tsdf, vol.weight, vol.color)]
    reset(); integrate(BATCH)
    identical = all(torch.equal(x, y) for x, y in zip(one, (vol.tsdf, vol.weight, vol.color)))
    del one
    verts, faces, _ = vol.extract()
    times = {"integrate_1": [], "integrate_%d" % BATCH: [], "extract": []}
    order = list(times)
    for r in range(args.rounds):
        for name in order[r % 3:] + order[:r % 3]:
            if name == "extract":
                ms, (verts, faces, _) = timed(vol.extract)
            else:
                reset()
                ms, _ = timed(lambda: integrate(1 if name == "integrate_1" else BATCH))
            times[name].append(ms)
    med = {k: float(np.median(v)) for k, v in times.items()}
    pix = V * H * W * (4 + 12)
    bytes_ = {"integrate_1": V * 40 * Ng + pix, "integrate_%d" % BATCH: (V // BATCH) * 40 * Ng + pix}
    gpu, power = card()
    out = {
        "workload": "%d views %dx%d depth+colour -> %d^3 coloured grid, %d surfels" % (V, W, H, NGRID, N_SURFELS),
        "gpu": gpu, "power_limit_w": power, "rounds": args.rounds,
        "ms": med, "spread_ms": {k: [float(min(v)), float(max(v))] for k, v in times.items()},
        "algorithmic_bytes": bytes_,
        "share_of_3.35TBps": {k: bytes_[k] / (med[k] * 1e-3) / PEAK_BPS for k in bytes_},
        "observed_points": int((vol.weight > 0).sum()), "verts": int(verts.shape[0]), "faces": int(faces.shape[0]),
        "batched_bit_identical": identical,
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
