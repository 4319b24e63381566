"""MCMC densification on the GPU against oracle/mcmc_oracle.py: the integer sampler id for id,
relocate and grow row by row (copies bit-exact, untouched rows bit-identical, relocation values
within 1 fp32 ulp, Adam moments zero exactly where specified), the noise displacement against fp64,
and a short training run that relocates, grows and injects noise."""
import numpy as np
import pytest
import torch

from oracle import mcmc_oracle as omc
from easygaussiansplatting_b200 import density
from easygaussiansplatting_b200.density import MCMCController
from easygaussiansplatting_b200.gau_io import adam_groups
from easygaussiansplatting_b200.scene import synthetic_scene

from test_gpu_parity import DEV, n, t

pytestmark = pytest.mark.gpu

WIDTHS = dict(pws=3, low_shs=3, high_shs=45, alphas_raw=1, scales_raw=3, rots_raw=4)


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def raw_alphas(N, seed, dead=0.05, nan=0):
    """alphas_raw [N, 1]: a `dead` fraction below logit(0.005), `nan` NaN rows, the rest live
    (with saturated ones at both ends)"""
    rng = np.random.default_rng(seed)
    a = rng.uniform(-5.0, 8.0, N).astype(np.float32)  # live: logit(0.005) = -5.29
    a[rng.random(N) < dead] = -7.0 - rng.random()
    if N > 8:
        a[rng.integers(0, N, 2)] = [30.0, 1e-3]
        a[rng.integers(0, N, 1)] = omc.alpha_raw_min()  # at the threshold: dead
    if nan:
        a[rng.choice(N, nan, replace=False)] = np.nan
    return a.reshape(N, 1)


def make_params(N, seed, alphas=None, extra=(), state=True):
    """six raw tensors (+ extra [N, D] at an odd 4-byte offset), an Adam with one real step"""
    rng = np.random.default_rng(seed + 7)
    raw = {k: rng.normal(size=(N, w)).astype(np.float32) for k, w in WIDTHS.items()}
    raw["scales_raw"] = (raw["scales_raw"] * 0.5 - 3).astype(np.float32)
    raw["alphas_raw"] = raw_alphas(N, seed) if alphas is None else alphas
    params = {k: torch.nn.Parameter(t(v)) for k, v in raw.items()}
    groups = adam_groups(params)
    for i, D in enumerate(extra):
        buf = torch.empty(N * D + 1, device=DEV)
        buf[1:] = t(rng.normal(size=N * D).astype(np.float32))
        params["f%d" % i] = torch.nn.Parameter(buf[1:].view(N, D))
        groups.append({"params": [params["f%d" % i]], "lr": 1e-2, "name": "f%d" % i})
    opt = torch.optim.Adam(groups, lr=1e-3)
    if state:
        for p in params.values():
            p.grad = torch.randn_like(p)
        opt.step()
        with torch.no_grad():
            params["alphas_raw"].copy_(t(raw["alphas_raw"]))  # the step must not revive or kill rows
    return params, opt


def snapshot(params, opt):
    p = {k: n(v).copy() for k, v in params.items()}
    st = [opt.state.get(v) for v in params.values()]
    if not st[0]:
        return p, None, None
    m = {k: n(opt.state[v]["exp_avg"]).copy() for k, v in params.items()}
    v_ = {k: n(opt.state[v]["exp_avg_sq"]).copy() for k, v in params.items()}
    return p, m, v_


def within_ulp(got, want, ulps=1):
    g = np.asarray(got, np.float32).view(np.int32).astype(np.int64)
    w = np.asarray(want, np.float32).view(np.int32).astype(np.int64)
    return np.abs(g - w).max(initial=0) <= ulps


# ---------------------------------------------------------------- 1. the sampler
@pytest.mark.parametrize("N", [1, 33, 1000, 1 << 20])
def test_sampler_ids_equal_the_oracle(N):
    for seed in range(3):
        a = raw_alphas(N, seed, nan=min(3, N - 1))
        ta = t(a).reshape(N)
        for mode, name in ((density.MCMC_RELOCATE, "relocate"), (density.MCMC_GROW, "grow")):
            w = omc.weights(a, name)
            total = int(w.sum(dtype=np.uint64))
            nd = len(omc.dead_rows(a))
            draws = max(nd, 1) if name == "relocate" else min(N, 5000) + 7
            ws, w_total, dead = density.mcmc_plan(ta, omc.alpha_raw_min(), mode, draws)
            assert w_total == total and (mode == density.MCMC_GROW or dead == nd), (N, seed, name)
            if total == 0:
                continue
            u = torch.rand(draws, dtype=torch.float64, device=DEV, generator=gen(seed))
            got = n(density.mcmc_sample(ws, N, u))
            assert np.array_equal(got, omc.sample(w, n(u))), (N, seed, name)


def test_sampler_equal_weights_and_edges():
    N = 1000
    a = np.full((N, 1), 1.5, np.float32)
    ws, total, dead = density.mcmc_plan(t(a).reshape(N), omc.alpha_raw_min(), density.MCMC_GROW, 20000)
    u = torch.rand(20000, dtype=torch.float64, device=DEV, generator=gen(3))
    got = n(density.mcmc_sample(ws, N, u))
    assert dead == 0 and np.array_equal(got, omc.sample(omc.weights(a, "grow"), n(u)))
    assert np.array_equal(got, np.floor(n(u) * N).astype(np.int64))  # equal weights: u N
    u = torch.tensor([0.0, np.nextafter(1.0, 0)], dtype=torch.float64, device=DEV)
    assert n(density.mcmc_sample(ws, N, u)).tolist() == [0, N - 1]
    ws, total, dead = density.mcmc_plan(torch.empty(0, device=DEV), 0.0, density.MCMC_RELOCATE, 0)
    assert (total, dead) == (0, 0)


# ---------------------------------------------------------------- 2. relocate
def check_relocate(N, seed, extra=(), state=True, alphas=None):
    params, opt = make_params(N, seed, alphas=alphas, extra=extra, state=state)
    ptrs = {k: v.data_ptr() for k, v in params.items()}
    p0, m0, v0 = snapshot(params, opt)
    nd = len(omc.dead_rows(p0["alphas_raw"]))
    u = n(torch.rand(max(nd, 1), dtype=torch.float64, device=DEV, generator=gen(seed)))
    ctl = MCMCController(cap_max=2 * N, verbose=False)
    rep = ctl.relocate(params, opt, generator=gen(seed), extra=["f%d" % i for i in range(len(extra))])
    p1, m1, v1 = snapshot(params, opt)
    assert all(params[k].data_ptr() == ptrs[k] for k in params)  # in place
    want, wm, wv, dead, sampled = omc.relocate(p0, m0, v0, u)
    assert rep == dict(relocated=len(sampled), total=N)
    touched = np.zeros(N, bool)
    touched[dead] = touched[sampled] = True
    for k in p1:
        assert np.array_equal(p1[k][~touched], p0[k][~touched], equal_nan=True), k  # untouched: bit-identical
        assert np.array_equal(p1[k][dead], p1[k][sampled]), k                     # copies: bit-exact
        if k not in ("alphas_raw", "scales_raw"):
            assert np.array_equal(p1[k][sampled], p0[k][sampled]), k
        else:
            assert within_ulp(p1[k][sampled], want[k][sampled]), k
    if m0 is not None:
        for got, before, exp in ((m1, m0, wm), (v1, v0, wv)):
            for k in got:
                assert np.array_equal(got[k], exp[k]), k  # zero exactly at sources and destinations
                assert not got[k][touched].any() and np.array_equal(got[k][~touched], before[k][~touched])
    for p in params.values():  # Adam keeps stepping on the same tensors
        p.grad = torch.randn_like(p)
    opt.step()
    assert all(torch.isfinite(p).all() for k, p in params.items() if k != "alphas_raw")
    return rep


@pytest.mark.parametrize("N,seed", [(33, 0), (1000, 1), (200001, 2)])
def test_relocate_vs_oracle(N, seed):
    rep = check_relocate(N, seed)
    assert rep["relocated"] > 0


def test_relocate_without_state_and_with_features():
    check_relocate(5000, 4, state=False)
    rep = check_relocate(5003, 5, extra=(1, 7, 32))
    assert rep["relocated"] > 0


def test_relocate_multiplicities_up_to_n_max():
    """one live row among many dead ones: hit c >> n_max times, r clamps at 51"""
    N = 300
    a = np.full((N, 1), -9.0, np.float32)
    a[[17, 200], 0] = [6.0, -4.0]
    rep = check_relocate(N, 6, alphas=a)
    assert rep["relocated"] == N - 2


def test_relocate_no_ops():
    for a, N in ((np.full((64, 1), -9.0, np.float32), 64), (np.full((64, 1), 2.0, np.float32), 64),
                 (np.zeros((0, 1), np.float32), 0)):
        params, opt = make_params(N, 8, alphas=a, state=N > 0)
        p0, m0, _ = snapshot(params, opt)
        rep = MCMCController(100, verbose=False).relocate(params, opt)
        assert rep == dict(relocated=0, total=N)
        p1, m1, _ = snapshot(params, opt)
        for k in p0:
            assert np.array_equal(p0[k], p1[k]) and (m0 is None or np.array_equal(m0[k], m1[k]))


# ---------------------------------------------------------------- 3. grow
def check_grow(N, cap, seed, extra=(), state=True, alphas=None, rate=0.05):
    params, opt = make_params(N, seed, alphas=alphas, extra=extra, state=state)
    p0, m0, v0 = snapshot(params, opt)
    n_add = omc.grow_count(N, cap, rate)
    u = n(torch.rand(max(n_add, 1), dtype=torch.float64, device=DEV, generator=gen(seed)))
    ctl = MCMCController(cap_max=cap, grow_rate=rate, verbose=False)
    old = dict(params)
    rep = ctl.grow(params, opt, generator=gen(seed), extra=["f%d" % i for i in range(len(extra))])
    assert rep == dict(added=n_add, total=N + n_add)
    if n_add == 0:
        assert all(params[k] is old[k] for k in params)
        return rep
    p1, m1, v1 = snapshot(params, opt)
    names = {g["name"]: g["params"][0] for g in opt.param_groups}
    assert all(names[k] is params[k] and params[k].shape[0] == N + n_add for k in params)
    want, wm, wv, sampled = omc.grow(p0, m0, v0, u, n_add)
    src = np.zeros(N, bool)
    src[sampled] = True
    for k in p1:
        assert np.array_equal(p1[k][:N][~src], p0[k][~src], equal_nan=True), k
        assert np.array_equal(p1[k][N:], p1[k][sampled]), k
        if k not in ("alphas_raw", "scales_raw"):
            assert np.array_equal(p1[k][sampled], p0[k][sampled]), k
        else:
            assert within_ulp(p1[k][sampled], want[k][sampled]), k
    if m0 is not None:
        for got, exp in ((m1, wm), (v1, wv)):
            for k in got:
                assert np.array_equal(got[k], exp[k]), k
    else:
        assert all(opt.state.get(p) is None for p in params.values())
    for p in params.values():
        p.grad = torch.randn_like(p)
    opt.step()
    return rep


@pytest.mark.parametrize("N,seed", [(1000, 10), (200003, 11)])
def test_grow_vs_oracle(N, seed):
    assert check_grow(N, 10 * N, seed)["added"] == int(N * 1.05) - N


def test_grow_without_state_and_with_features():
    check_grow(4000, 10 ** 6, 12, state=False)
    check_grow(4001, 10 ** 6, 13, extra=(1, 7, 32))


def test_grow_cap_edges_and_nan_rows():
    assert check_grow(1000, 1000, 14)["added"] == 0      # N >= cap: no-op
    assert check_grow(1000, 900, 14)["added"] == 0
    assert check_grow(1000, 1013, 15)["added"] == 13     # clipped to cap - N
    assert check_grow(19, 100, 16)["added"] == 0         # int(0.05 N) = 0
    a = raw_alphas(500, 17, nan=40)
    assert check_grow(500, 10 ** 4, 17, alphas=a, rate=0.5)["added"] == 250  # NaN rows are never sources
    a = np.full((50, 1), np.nan, np.float32)
    params, opt = make_params(50, 18, alphas=a)
    assert MCMCController(100, grow_rate=0.5, verbose=False).grow(params, opt) == dict(added=0, total=50)


# ---------------------------------------------------------------- 4. noise
def test_inject_noise_vs_fp64():
    N = 100000
    params, opt = make_params(N, 20, state=False)
    rng = np.random.default_rng(20)
    with torch.no_grad():
        params["pws"].zero_()  # the update itself is the displacement (no rounding against |pws|)
        a = rng.normal(size=N).astype(np.float32) * 4
        a[:1000], a[1000:2000], a[2000:3000] = -30.0, 30.0, np.float32(np.log(0.995 / 0.005))  # gate ends, middle
        params["alphas_raw"].copy_(t(a.reshape(N, 1)))
        s = params["scales_raw"]
        s.copy_(t(rng.uniform(-3.3, -2.7, size=(N, 3)).astype(np.float32)))
        s[3000:3100] = -float("inf")   # zero scales
        q = params["rots_raw"]
        q.mul_(t(np.exp(rng.uniform(-3, 3, size=(N, 1))).astype(np.float32)))  # unnormalised
        q[3100:3110] = 0.0
    for g in opt.param_groups:
        if g["name"] == "pws":
            g["lr"] = 1.6e-4
    p0, _, _ = snapshot(params, opt)
    ptr = params["pws"].data_ptr()
    z = MCMCController(10 ** 6, verbose=False).inject_noise(params, opt, generator=gen(20))
    assert params["pws"].data_ptr() == ptr
    got = n(params["pws"]).astype(np.float64)
    want = omc.noise(p0, n(z), 1.6e-4)
    row = np.abs(want).max(axis=1, keepdims=True)
    assert np.all(np.abs(got - want) <= 1e-5 * row + 1e-30), float((np.abs(got - want) / np.maximum(row, 1e-30)).max())
    assert not got[3000:3100].any() and np.abs(got[1000:2000]).max() < 1e-30
    assert (np.abs(got[:1000]).max(axis=1) > 0).all() and (np.abs(got[2000:3000]).max(axis=1) > 0).all()


# ---------------------------------------------------------------- 5. training
def _train(features):
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused, GSFunctionFusedFeatures
    W, H, N = 160, 120, 6000
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=30)
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]))
    gt = {k: t(sc[k]) for k in ("pws", "shs", "alphas", "scales", "rots")}
    us0 = torch.zeros((N, 2), device=DEV)
    D = 4
    labels = torch.nn.functional.one_hot(torch.from_numpy(np.random.default_rng(1).integers(0, D, N)), D).float().to(DEV)
    with torch.no_grad():
        target, _ = GSFunctionFused.apply(gt["pws"], gt["shs"], gt["alphas"][:, None], gt["scales"], gt["rots"], us0, cam)
        if features:
            ftarget = GSFunctionFusedFeatures.apply(gt["pws"], gt["shs"], gt["alphas"][:, None], gt["scales"],
                                                    gt["rots"], us0, labels, cam)[1]
    N0 = 3000  # start from half the Gaussians, perturbed, with some nearly transparent
    rng = np.random.default_rng(31)
    a0 = np.log(sc["alphas"][:N0] / (1 - sc["alphas"][:N0])).astype(np.float32)
    a0[rng.random(N0) < 0.1] = -8.0
    raw = dict(pws=sc["pws"][:N0] + rng.normal(size=(N0, 3)).astype(np.float32) * 0.02, low_shs=np.zeros((N0, 3), np.float32),
               high_shs=np.zeros((N0, 45), np.float32), alphas_raw=a0.reshape(N0, 1),
               scales_raw=np.log(sc["scales"][:N0]), rots_raw=sc["rots"][:N0])
    params = {k: torch.nn.Parameter(t(np.ascontiguousarray(v, dtype=np.float32))) for k, v in raw.items()}
    groups = adam_groups(params)
    extra = ()
    if features:
        params["features"] = torch.nn.Parameter(torch.full((N0, D), 1.0 / D, device=DEV))
        groups.append({"params": [params["features"]], "lr": 0.05, "name": "features"})
        extra = ("features",)
    for g in groups:
        g["lr"] = dict(pws=1.6e-4, low_shs=0.02).get(g["name"], g["lr"])
    opt = torch.optim.Adam(groups, lr=1e-3)
    cap = 4000
    ctl = MCMCController(cap, grow_rate=0.1, noise_lr=1e3, verbose=False)
    rng_t = gen(32)
    losses = []
    for step in range(80):
        P = params
        alphas = torch.sigmoid(P["alphas_raw"])
        scales = torch.exp(P["scales_raw"])
        rots = torch.nn.functional.normalize(P["rots_raw"], dim=1)
        shs = torch.cat([P["low_shs"], P["high_shs"][:, :9]], dim=1)
        us = torch.zeros((P["pws"].shape[0], 2), device=DEV, requires_grad=True)
        if features:
            img, fmap, _ = GSFunctionFusedFeatures.apply(P["pws"], shs, alphas, scales, rots, us, P["features"], cam)
            loss = ((img - target) ** 2).mean() + ((fmap - ftarget) ** 2).mean()
        else:
            img, _ = GSFunctionFused.apply(P["pws"], shs, alphas, scales, rots, us, cam)
            loss = ((img - target) ** 2).mean()
        loss = loss + 0.01 * alphas.mean() + 0.01 * scales.mean()  # the paper's two regularisers
        opt.zero_grad()
        loss.backward()
        opt.step()
        ctl.inject_noise(params, opt, generator=rng_t)
        losses.append(float(loss.detach()))
        if step % 10 == 9:
            ctl.relocate(params, opt, generator=rng_t, extra=extra)
            ctl.grow(params, opt, generator=rng_t, extra=extra)
        assert params["pws"].shape[0] <= cap
        assert all(torch.isfinite(p).all() for p in params.values())
    assert params["pws"].shape[0] == cap
    assert np.mean(losses[-5:]) < 0.7 * np.mean(losses[:5]), losses[::10]


def test_training_with_mcmc():
    _train(features=False)


def test_training_with_mcmc_and_features():
    _train(features=True)
