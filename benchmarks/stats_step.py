"""Cost of the contribution statistics at BASELINE config 2 (1M Gaussians, SH degree 3, 1920x1080).

- The kernels: CUDA-event times (gsb_profile_*) of draw_stats, the replay, next to draw, the colour
  forward it replays.
- The replay against the workaround it replaces: `splat_stats` (records given) against
  `splatB_features` with features = ones[N, 1] and dL/dF = 1, whose dL/dfeatures is sum_p w; the two
  alternate in rounds, in the same process, so that clock and thermal drift hit both alike.
- The masked prune: `density.prune` of a 1M-row model with Adam moments (40 % dropped) against the
  torch chain it replaces (t[keep] for the six tensors and both moments of each).
Medians over rounds, with the card's name and power limit read in the same run.  Prints one JSON line.

    python benchmarks/stats_step.py [--rounds 7] [--steps 10]
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
from easygaussiansplatting_b200.density import prune  # noqa: E402
from easygaussiansplatting_b200.gau_io import adam_groups  # noqa: E402
from easygaussiansplatting_b200.scene import synthetic_scene  # noqa: E402

N, W, H, SH = 1_000_000, 1920, 1080, 48
KERNELS = ("draw", "draw_stats")
WIDTHS = dict(pws=3, low_shs=3, high_shs=45, alphas_raw=1, scales_raw=3, rots_raw=4)


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
    C_d, C_ll = ctypes.c_double, ctypes.c_longlong
    sc = synthetic_scene(N, W, H, sh_dim=SH, seed=0)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    al = T(sc["alphas"])
    us, ci, col, d, ar, recs = ops.preprocess(*[T(sc[k]) for k in ("pws", "rots", "scales", "shs", "Rcw", "tcw", "twc")],
                                              sc["fx"], sc["fy"], sc["cx"], sc["cy"], W, H, alphas=al)
    frame = ops.splat(H, W, us, ci, al, d, col, ar, records=recs)
    contrib, final_tau, ranges, gsid = frame[1:5]
    ones, dl_ones = torch.ones((N, 1), device=dev), torch.ones((1, H, W), device=dev)

    def replay():
        ops.splat_stats(H, W, contrib, ranges, gsid, records=recs)

    def workaround():
        ops.splatB_features(H, W, ones, contrib, final_tau, ranges, gsid, dl_ones, records=recs)

    def draw():
        ops.splat(H, W, us, ci, al, d, col, ar, records=recs)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

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

    # the two results agree (fp32 atomic order) before anything is timed
    ws = ops.splat_stats(H, W, contrib, ranges, gsid, records=recs)[0]
    df = ops.splatB_features(H, W, ones, contrib, final_tau, ranges, gsid, dl_ones, records=recs)[1][:, 0]
    agree = float((ws - df).abs().max()) / float(ws.abs().max())

    gpu, power = card()
    for fn in (replay, workaround, draw):  # warm-up
        for _ in range(3):
            fn()
    res = {"replay_ms": [], "workaround_ms": [], "draw_stats_kernel_ms": [], "draw_kernel_ms": []}
    for r in range(args.rounds):
        order = (replay, workaround) if r % 2 == 0 else (workaround, replay)
        for fn in order:
            res["replay_ms" if fn is replay else "workaround_ms"].append(timed(fn))
        res["draw_stats_kernel_ms"].append(kernel_ms(replay, "draw_stats"))
        res["draw_kernel_ms"].append(kernel_ms(draw, "draw"))
    del frame, contrib, final_tau, ranges, gsid, recs, us, ci, col, d, ar, ones, dl_ones
    torch.cuda.empty_cache()

    # the masked prune at 1M rows with Adam moments
    rng = np.random.default_rng(2)
    base = {k: T(rng.normal(size=(N, w)).astype(np.float32)) for k, w in WIDTHS.items()}
    keep = T(rng.uniform(size=N) < 0.6)

    def model():
        params = {k: v.clone().requires_grad_() for k, v in base.items()}
        opt = torch.optim.Adam(adam_groups(params), lr=1e-3)
        for p in params.values():
            opt.state[p] = {"step": torch.tensor(1.0), "exp_avg": 0.5 * p.detach(), "exp_avg_sq": p.detach().abs()}
        return params, opt

    def torch_chain(params, opt):
        for g in opt.param_groups:
            old = g["params"][0]
            st = opt.state.pop(old)
            new = torch.nn.Parameter(old.detach()[keep].requires_grad_(True))
            st["exp_avg"], st["exp_avg_sq"] = st["exp_avg"][keep], st["exp_avg_sq"][keep]
            opt.state[new] = st
            g["params"][0] = new
            params[g["name"]] = new

    def one(fn):
        params, opt = model()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn(params, opt)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), params, opt

    lib_prune = lambda p, o: prune(p, o, keep, verbose=False)  # noqa: E731
    _, pa, oa = one(lib_prune)
    _, pb, ob = one(torch_chain)
    same = all(torch.equal(pa[k], pb[k]) for k in WIDTHS) and all(
        torch.equal(oa.state[pa[k]][m], ob.state[pb[k]][m]) for k in WIDTHS for m in ("exp_avg", "exp_avg_sq"))
    del pa, oa, pb, ob
    for _ in range(2):
        one(lib_prune), one(torch_chain)
    res["prune_ms"], res["torch_chain_ms"] = [], []
    for r in range(args.rounds):
        order = (lib_prune, torch_chain) if r % 2 == 0 else (torch_chain, lib_prune)
        for fn in order:
            res["prune_ms" if fn is lib_prune else "torch_chain_ms"].append(one(fn)[0])

    med = {k: float(np.median(v)) for k, v in res.items()}
    out = {"gpu": gpu, "power_limit_w": power, "config": "N=%d %dx%d SH degree 3" % (N, W, H),
           "rounds": args.rounds, "steps_per_round": args.steps,
           "ms": {k: round(v, 4) for k, v in med.items()},
           "spread_ms": {k: round(float(np.max(v) - np.min(v)), 4) for k, v in res.items()},
           "replay_vs_workaround": round(med["replay_ms"] / med["workaround_ms"], 4),
           "draw_stats_vs_draw": round(med["draw_stats_kernel_ms"] / med["draw_kernel_ms"], 4),
           "prune_vs_torch_chain": round(med["prune_ms"] / med["torch_chain_ms"], 4),
           "weight_sum_vs_workaround_rel_err": agree, "prune_equals_torch_chain": bool(same)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
