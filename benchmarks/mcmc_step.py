"""Cost of MCMC densification at N = 1M Gaussians (DESIGN 3.11).

Times the three MCMCController operations against the same operations composed from torch
(torch.multinomial, bincount, boolean / index writes into the 18 tensors, a bmm of [N,3,3]
covariances), the two alternating in rounds so that clock drift hits both alike:
  noise     inject_noise on all N rows;
  relocate  5 % dead rows moved onto live ones (the state is restored between calls, untimed);
  grow      1M -> 1.05M rows (fresh tensors each call, rebuilt untimed).
Each time is CUDA events around the call (host syncs included); the MCMC kernels' own time comes
from the library's per-kernel events.  Achieved bytes/s = the algorithmic bytes over the kernel
time.  Medians over rounds, with the card's name and power limit read in the same run.  Prints
one JSON line.

    python benchmarks/mcmc_step.py [--rounds 7] [--n 1000000]
"""
import argparse
import ctypes
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from easygaussiansplatting_b200 import _lib  # noqa: E402
from easygaussiansplatting_b200.density import MCMCController  # noqa: E402
from easygaussiansplatting_b200.gau_io import adam_groups  # noqa: E402

WIDTHS = dict(pws=3, low_shs=3, high_shs=45, alphas_raw=1, scales_raw=3, rots_raw=4)
ROW = 4 * sum(WIDTHS.values())  # 236 B: one Gaussian's six tensors
KERNELS = ("mcmc_scan", "mcmc_sample", "mcmc_relocate", "mcmc_grow", "mcmc_noise")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(q.splitlines()[0])
    except Exception:
        power = None
    return name, power


def algorithmic_bytes(N, n_reloc, n_grow):
    """plan: alphas read twice, W (8 B) and the hit count (4 B) written; relocate: n source rows
    read and n destination rows written, the moments of 2n rows zeroed; grow: every row and both
    moments read and written once, n new rows read from their source and written with moments"""
    plan = N * (8 + 8 + 4)
    return dict(noise=68 * N, relocate=plan + n_reloc * (2 * ROW + 2 * 2 * ROW),
                grow=plan + 2 * 3 * ROW * N + n_grow * (ROW + 3 * ROW))


# ---------------------------------------------------------------- the torch composition
def torch_relocation(o, s, ratios, binoms, min_opacity, n_max):
    """the relocation value in fp32 torch: the alternating series over a binomial table, [n, n_max]"""
    r = torch.clamp(ratios, 1, n_max).long()
    op = torch.clamp(1.0 - (1.0 - o) ** (1.0 / r), min_opacity, 1.0 - torch.finfo(torch.float32).eps)
    m = torch.arange(1, n_max + 1, device=o.device)
    sign = 1.0 - 2.0 * ((m + 1) % 2)
    terms = binoms[r][:, 1:] * sign * op[:, None] ** m / torch.sqrt(m.float())
    denom = (terms * (m[None, :] <= r[:, None])).sum(1)
    return op, s * (o / denom)[:, None]


def torch_relocate(P, M, V, min_opacity, n_max, binoms):
    a = P["alphas_raw"][:, 0]
    thr = math.log(min_opacity / (1 - min_opacity))
    dead = ~(a > thr)
    dead_idx = dead.nonzero()[:, 0]
    n = dead_idx.numel()
    if n == 0:
        return 0
    probs = torch.sigmoid(a) * (~dead)
    sampled = torch.multinomial(probs, n, replacement=True)
    ratios = torch.bincount(sampled, minlength=a.shape[0])[sampled] + 1
    o = torch.sigmoid(a[sampled])
    op, s = torch_relocation(o, torch.exp(P["scales_raw"][sampled]), ratios.float(), binoms, min_opacity, n_max)
    P["alphas_raw"][sampled, 0] = torch.logit(op)
    P["scales_raw"][sampled] = torch.log(s)
    for k in P:
        P[k][dead_idx] = P[k][sampled]
        for d in (M, V):
            d[k][sampled] = 0
            d[k][dead_idx] = 0
    return n


def torch_grow(P, M, V, n, min_opacity, n_max, binoms):
    a = P["alphas_raw"][:, 0]
    sampled = torch.multinomial(torch.sigmoid(a), n, replacement=True)
    ratios = torch.bincount(sampled, minlength=a.shape[0])[sampled] + 1
    o = torch.sigmoid(a[sampled])
    op, s = torch_relocation(o, torch.exp(P["scales_raw"][sampled]), ratios.float(), binoms, min_opacity, n_max)
    P["alphas_raw"][sampled, 0] = torch.logit(op)
    P["scales_raw"][sampled] = torch.log(s)
    out = {}
    for k in P:
        out[k] = torch.cat([P[k], P[k][sampled]])
        for d in (M, V):
            d[k][sampled] = 0
            d[k] = torch.cat([d[k], torch.zeros((n,) + d[k].shape[1:], device=d[k].device)])
    return out


def torch_noise(P, lr, noise_lr, z):
    q = torch.nn.functional.normalize(P["rots_raw"], dim=1)
    w, x, y, zq = q.unbind(1)
    R = torch.stack([1 - 2 * (y * y + zq * zq), 2 * (x * y - zq * w), 2 * (x * zq + y * w),
                     2 * (x * y + zq * w), 1 - 2 * (x * x + zq * zq), 2 * (y * zq - x * w),
                     2 * (x * zq - y * w), 2 * (y * zq + x * w), 1 - 2 * (x * x + y * y)], 1).view(-1, 3, 3)
    M = R * torch.exp(P["scales_raw"])[:, None, :]
    cov = torch.bmm(M, M.transpose(1, 2))
    o = torch.sigmoid(P["alphas_raw"])
    gate = torch.sigmoid(100.0 * ((1 - o) - 0.995))
    P["pws"] += torch.bmm(cov, z[:, :, None])[:, :, 0] * lr * noise_lr * gate


# ---------------------------------------------------------------- the run
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--n", type=int, default=1_000_000)
    args = ap.parse_args()
    N = args.n
    dev = torch.device("cuda", 0)
    lib = _lib.load()
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    kid = {k: names.index(k) for k in KERNELS}
    C_d, C_ll = ctypes.c_double, ctypes.c_longlong
    rng = np.random.default_rng(0)
    base = {k: torch.from_numpy(rng.normal(size=(N, w)).astype(np.float32)).to(dev) for k, w in WIDTHS.items()}
    base["scales_raw"] = base["scales_raw"] * 0.5 - 4
    a = rng.uniform(-4.0, 6.0, N).astype(np.float32)
    a[rng.random(N) < 0.05] = -8.0  # 5 % dead
    base["alphas_raw"] = torch.from_numpy(a.reshape(N, 1)).to(dev)
    mom = {k: torch.rand_like(v) for k, v in base.items()}
    n_dead = int((a <= np.float32(math.log(0.005 / 0.995))).sum())
    n_grow = int(N * 1.05) - N
    ctl = MCMCController(cap_max=10 * N, verbose=False)

    def fresh():
        params = {k: torch.nn.Parameter(v.clone()) for k, v in base.items()}
        opt = torch.optim.Adam(adam_groups(params), lr=1e-3)
        for k, p in params.items():
            opt.state[p] = {"step": torch.tensor(1.0), "exp_avg": mom[k].clone(), "exp_avg_sq": mom[k].clone()}
        for g in opt.param_groups:
            if g["name"] == "pws":
                g["lr"] = 1.6e-4
        return params, opt

    def fresh_torch():
        P = {k: v.clone() for k, v in base.items()}
        return P, {k: m.clone() for k, m in mom.items()}, {k: m.clone() for k, m in mom.items()}

    binoms = torch.tensor([[math.comb(r, k) for k in range(ctl.n_max + 1)] for r in range(ctl.n_max + 1)],
                          dtype=torch.float32, device=dev)  # C(r, k)
    gen = torch.Generator(device=dev).manual_seed(0)

    def timed(setup, fn):
        state = setup()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn(state)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    ops = {
        "noise": (fresh, lambda s: ctl.inject_noise(s[0], s[1], generator=gen),
                  fresh_torch, lambda s: torch_noise(s[0], 1.6e-4, ctl.noise_lr, torch.randn((N, 3), device=dev))),
        "relocate": (fresh, lambda s: ctl.relocate(s[0], s[1], generator=gen),
                     fresh_torch, lambda s: torch_relocate(s[0], s[1], s[2], ctl.min_opacity, ctl.n_max, binoms)),
        "grow": (fresh, lambda s: ctl.grow(s[0], s[1], generator=gen),
                 fresh_torch, lambda s: torch_grow(s[0], s[1], s[2], n_grow, ctl.min_opacity, ctl.n_max, binoms)),
    }
    res = {op: {"native_ms": [], "torch_ms": [], "kernel_ms": []} for op in ops}
    for op, (setup, fn, setup_t, fn_t) in ops.items():  # warm-up
        for _ in range(2):
            timed(setup, fn)
            timed(setup_t, fn_t)
    for r in range(args.rounds):
        for op, (setup, fn, setup_t, fn_t) in ops.items():
            pair = ((setup, fn, "native_ms"), (setup_t, fn_t, "torch_ms"))
            for s, f, key in (pair if r % 2 == 0 else pair[::-1]):
                res[op][key].append(timed(s, f))
            # kernel time of the native call: the library's per-kernel events over one more call
            state = setup()
            torch.cuda.synchronize()
            lib.gsb_profile_enable(1)
            for k in kid.values():
                lib.gsb_profile_read(k, ctypes.byref(C_d()), ctypes.byref(C_ll()))
            fn(state)
            torch.cuda.synchronize()
            lib.gsb_profile_enable(0)
            tot = 0.0
            for k in kid.values():
                ms, cnt = C_d(), C_ll()
                lib.gsb_profile_read(k, ctypes.byref(ms), ctypes.byref(cnt))
                tot += ms.value
            res[op]["kernel_ms"].append(tot)
    gpu, power = card()
    nbytes = algorithmic_bytes(N, n_dead, n_grow)
    out = {"gpu": gpu, "power_limit_w": power, "N": N, "dead": n_dead, "grown": n_grow, "rounds": args.rounds,
           "ops": {}}
    for op, d in res.items():
        med = {k: float(np.median(v)) for k, v in d.items()}
        out["ops"][op] = {
            "ms": {k: round(v, 4) for k, v in med.items()},
            "spread_ms": {k: round(float(np.max(v) - np.min(v)), 4) for k, v in d.items()},
            "torch_over_native": round(med["torch_ms"] / med["native_ms"], 2),
            "algorithmic_bytes": nbytes[op],
            "kernel_gb_per_s": round(nbytes[op] / (med["kernel_ms"] * 1e-3) / 1e9, 1),
            "datasheet_bound_ms": round(nbytes[op] / 3.35e12 * 1e3, 4),
        }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
