"""GaussianAdam on the GPU: dense steps against torch.optim.Adam (foreach) and the fp64 oracle,
selective steps row by row, state_dict interchange in both directions, the density and MCMC
controllers on a GaussianAdam, the safety of the fused classes' visibility mask, and short training
runs.

Tolerances.  Against torch (both fp32, the same operations): m and v within 2 fp32 ulp per element,
p within 2 ulp(p) + 1e-6 |dp| with dp torch's change of p over the run.  Against the oracle (one
step from the kernel's own fp32 state): v within 2 ulp; m within 4 ulp of its larger term
max(beta1 |m|, (1 - beta1) |g|) (the sum may cancel); p within 2 ulp(p) + 1e-6 |dp| plus the part of
m's allowance the step carries into p."""
import copy

import numpy as np
import pytest
import torch

from oracle import adam_oracle as oad
from easygaussiansplatting_b200.density import DensityController, MCMCController
from easygaussiansplatting_b200.gau_io import adam_groups
from easygaussiansplatting_b200.optim import GaussianAdam

from test_gpu_parity import DEV, n, t

pytestmark = pytest.mark.gpu

WIDTHS = dict(pws=3, low_shs=3, high_shs=45, alphas_raw=1, scales_raw=3, rots_raw=4)
EXTRA_D = (1, 7, 16, 45, 64)
B1, B2 = 0.9, 0.999


def ulp(x):
    return np.spacing(np.abs(np.asarray(x, np.float32))).astype(np.float64)


def ulp_dist(a, b):
    """distance in fp32 ulps (monotone integer map of the bit patterns)"""
    def key(x):
        i = np.asarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(key(a) - key(b))


def make_tensors(N, seed):
    """the six reference widths, extras [N, D] for D in EXTRA_D, and a [N, 7] view at an odd float offset"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    out = {k: torch.randn((N, w), device=DEV, generator=g) for k, w in WIDTHS.items()}
    for D in EXTRA_D:
        out["x%d" % D] = torch.randn((N, D), device=DEV, generator=g)
    buf = torch.randn(N * 7 + 3, device=DEV, generator=g)
    out["odd"] = buf[1:N * 7 + 1].view(N, 7)
    return out


def clone_params(src):
    """leaf Parameters with src's values at the same float offset mod 4 as src"""
    out = {}
    for k, x in src.items():
        off = x.storage_offset() % 4
        buf = torch.empty(x.numel() + 4, device=DEV)
        v = buf[off:off + x.numel()].view(x.shape)
        v.copy_(x)
        out[k] = torch.nn.Parameter(v)
    return out


def groups_of(params, lrs):
    return [{"params": [params[k]], "lr": lrs[k], "name": k} for k in params]


def lrs_for(names):
    lrs = {k: 1e-3 * (1 + i) for i, k in enumerate(names)}
    lrs["low_shs"] = 0.0  # an lr = 0 group
    lrs["x16"] = 0.05
    return lrs


def grads_for(params, seed, step, none=()):
    g = torch.Generator(device=DEV).manual_seed(seed * 1000 + step)
    out = {}
    for k, p in params.items():
        if k in none:
            out[k] = None
            continue
        scale = float(torch.empty(1).uniform_(-6, 1, generator=torch.Generator().manual_seed(seed + step)).exp())
        out[k] = torch.randn(p.shape, device=DEV, generator=g) * scale
    return out


def set_grads(params, grads):
    for k, p in params.items():
        p.grad = None if grads[k] is None else grads[k].clone()


def state_np(params, opt):
    return {k: (n(p).copy(), n(opt.state[p]["exp_avg"]).copy(), n(opt.state[p]["exp_avg_sq"]).copy(),
                float(opt.state[p]["step"])) for k, p in params.items() if p in opt.state}


def check_vs_torch(ours, ref, start):
    """ours / ref: dicts of (p, m, v, step) after the run; start: the params before it"""
    assert ours.keys() == ref.keys()
    for k in ours:
        (p, m, v, s), (pr, mr, vr, sr) = ours[k], ref[k]
        assert s == sr, k
        assert ulp_dist(m, mr).max(initial=0) <= 2, (k, ulp_dist(m, mr).max())
        assert ulp_dist(v, vr).max(initial=0) <= 2, (k, ulp_dist(v, vr).max())
        tol = 2 * ulp(pr) + 1e-6 * np.abs(pr.astype(np.float64) - start[k])
        err = np.abs(p.astype(np.float64) - pr)
        assert (err <= tol).all(), (k, float((err - tol).max()))


def check_vs_oracle(before, after, grads, lrs, eps, vis=None):
    """one step: `before` (p, m, v, step) -> `after`, against oracle.adam_step in fp64"""
    for k, (p0, m0, v0, s0) in before.items():
        if grads[k] is None:
            assert np.array_equal(after[k][0], p0) and after[k][3] == s0, k
            continue
        g = n(grads[k])
        pr, mr, vr, sr = oad.adam_step(p0, g, m0, v0, s0, lrs[k], B1, B2, eps, visibility=vis)
        p, m, v, s = after[k]
        assert s == sr, k
        big = np.maximum(B1 * np.abs(m0.astype(np.float64)), (1 - B1) * np.abs(g.astype(np.float64)))
        m_tol = 4 * ulp(big)
        assert (np.abs(m - mr) <= m_tol).all(), (k, float((np.abs(m - mr) - m_tol).max()))
        assert (np.abs(v - vr) <= 2 * ulp(vr)).all(), k
        denom = np.sqrt(vr) / np.sqrt(1 - B2 ** sr) + eps
        step = lrs[k] / (1 - B1 ** sr)
        p_tol = 2 * ulp(pr) + 1e-6 * np.abs(pr - p0) + step * m_tol / denom
        assert (np.abs(p - pr) <= p_tol).all(), (k, float((np.abs(p - pr) - p_tol).max()))


# ---------------------------------------------------------------- 1. dense
@pytest.mark.parametrize("N", [0, 1, 31, 1000, 1_000_003])
def test_dense_matches_torch_foreach_and_the_oracle(N):
    src = make_tensors(N, seed=N + 1)
    ours, ref = clone_params(src), clone_params(src)
    assert N == 0 or ours["odd"].data_ptr() % 16 != 0  # the scalar head / tail path
    lrs = lrs_for(src)
    eps = 1e-15
    opt = GaussianAdam(groups_of(ours, lrs), eps=eps)
    opt_ref = torch.optim.Adam(groups_of(ref, lrs), eps=eps)
    assert opt_ref.defaults["foreach"] is None and opt_ref.defaults["fused"] is None  # torch picks foreach
    start = {k: n(x).astype(np.float64) for k, x in src.items()}
    small = N <= 1000
    for step in range(20):
        grads = grads_for(src, N, step, none=("x7",) if step % 3 == 1 else ())  # a group with grad None
        set_grads(ours, grads)
        set_grads(ref, grads)
        before = state_np(ours, opt) if (small or step == 19) and step > 0 else None
        opt.step()
        opt_ref.step()
        if before is not None:
            check_vs_oracle(before, state_np(ours, opt), grads, lrs, eps)
    assert float(opt.state[ours["x7"]]["step"]) == 20 - 7  # skipped steps do not count
    check_vs_torch(state_np(ours, opt), state_np(ref, opt_ref), start)
    assert np.array_equal(n(ours["low_shs"]), n(src["low_shs"]))  # lr = 0


def test_dense_betas_eps_and_closure():
    """other betas (both lerp branches of torch) and eps, a closure, and one launch per step"""
    from easygaussiansplatting_b200 import _lib
    lib = _lib.load()
    kid = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())].index("adam")
    for betas, eps in (((0.3, 0.5), 1e-3), ((0.0, 0.99), 1e-8), ((0.6, 0.9), 1e-6)):
        src = make_tensors(257, seed=3)
        ours, ref = clone_params(src), clone_params(src)
        lrs = lrs_for(src)
        opt = GaussianAdam(groups_of(ours, lrs), betas=betas, eps=eps)
        opt_ref = torch.optim.Adam(groups_of(ref, lrs), betas=betas, eps=eps)
        start = {k: n(x).astype(np.float64) for k, x in src.items()}
        for step in range(10):
            grads = grads_for(src, 9, step)
            set_grads(ours, grads)
            set_grads(ref, grads)
            before = lib.gsb_profile_launches(kid)
            assert opt.step(closure=lambda: 1.5) == 1.5
            assert lib.gsb_profile_launches(kid) == before + 1
            opt_ref.step()
        check_vs_torch(state_np(ours, opt), state_np(ref, opt_ref), start)


def test_refusals():
    p = torch.nn.Parameter(torch.zeros((4, 3), device=DEV))
    for kw in (dict(amsgrad=True), dict(weight_decay=1e-2), dict(maximize=True), dict(capturable=True)):
        with pytest.raises(ValueError):
            GaussianAdam([p], **kw)
    with pytest.raises(ValueError):
        GaussianAdam([torch.nn.Parameter(torch.zeros(4, 3))])  # CPU
    with pytest.raises(ValueError):
        GaussianAdam([torch.nn.Parameter(torch.zeros((4, 3), device=DEV, dtype=torch.float64))])
    with pytest.raises(ValueError):
        GaussianAdam([torch.nn.Parameter(torch.zeros((3, 4), device=DEV).t())])  # non-contiguous


# ---------------------------------------------------------------- 2. selective
@pytest.mark.parametrize("N", [1, 31, 1000, 1_000_003])
def test_selective_random_masks(N):
    src = make_tensors(N, seed=7 + N)
    ours = clone_params(src)
    lrs = lrs_for(src)
    eps = 1e-15
    opt = GaussianAdam(groups_of(ours, lrs), eps=eps)
    gen = torch.Generator(device=DEV).manual_seed(N)
    for step in range(6):
        grads = grads_for(src, 2 * N, step)
        set_grads(ours, grads)
        vis = torch.rand(N, device=DEV, generator=gen) < 0.5
        if step % 2:
            vis = vis.to(torch.uint8)
        before = state_np(ours, opt) if step else {k: (n(p).copy(), np.zeros(p.shape, np.float32),
                                                       np.zeros(p.shape, np.float32), 0.0) for k, p in ours.items()}
        opt.step(visibility=vis)
        after = state_np(ours, opt)
        hid = ~n(vis).astype(bool)
        for k in before:
            for i in range(3):
                assert np.array_equal(after[k][i][hid].view(np.int32), before[k][i][hid].view(np.int32)), (k, i)
        if N <= 1000 or step == 5:
            check_vs_oracle(before, after, grads, lrs, eps, vis=n(vis).astype(bool))


def test_selective_all_true_is_dense_and_all_false_only_counts():
    N = 4099
    src = make_tensors(N, seed=11)
    a, b, c = clone_params(src), clone_params(src), clone_params(src)
    lrs = lrs_for(src)
    oa, ob, oc = (GaussianAdam(groups_of(x, lrs), eps=1e-15) for x in (a, b, c))
    for step in range(4):
        grads = grads_for(src, 5, step)
        for x in (a, b, c):
            set_grads(x, grads)
        oa.step()
        ob.step(visibility=torch.ones(N, dtype=torch.bool, device=DEV))
        if step < 2:
            oc.step()
    sa, sb = state_np(a, oa), state_np(b, ob)
    for k in sa:
        for i in range(3):
            assert np.array_equal(sa[k][i].view(np.int32), sb[k][i].view(np.int32)), (k, i)
    before = state_np(c, oc)
    oc.step(visibility=torch.zeros(N, dtype=torch.uint8, device=DEV))
    after = state_np(c, oc)
    for k in before:
        assert after[k][3] == before[k][3] + 1
        for i in range(3):
            assert np.array_equal(after[k][i].view(np.int32), before[k][i].view(np.int32)), (k, i)


def test_selective_refusals():
    N = 64
    p = torch.nn.Parameter(torch.zeros((N, 3), device=DEV))
    q = torch.nn.Parameter(torch.zeros(N, device=DEV))
    opt = GaussianAdam([p])
    p.grad = torch.ones_like(p)
    for bad in (torch.ones(N + 1, dtype=torch.bool, device=DEV), torch.ones(N, dtype=torch.float32, device=DEV),
                torch.ones(N, dtype=torch.bool), torch.ones((N, 1), dtype=torch.bool, device=DEV)):
        with pytest.raises(ValueError):
            opt.step(visibility=bad)
    opt2 = GaussianAdam([q])
    q.grad = torch.ones_like(q)
    with pytest.raises(ValueError):  # selective steps take [N, D] params
        opt2.step(visibility=torch.ones(N, dtype=torch.bool, device=DEV))


# ---------------------------------------------------------------- 3. interchange
@pytest.mark.parametrize("first", ["ours", "torch"])
def test_state_dict_interchange(first):
    N = 3001
    src = make_tensors(N, seed=21)
    lrs = lrs_for(src)
    make = {"ours": lambda g: GaussianAdam(g, eps=1e-15), "torch": lambda g: torch.optim.Adam(g, eps=1e-15)}
    second = "torch" if first == "ours" else "ours"
    a, b = clone_params(src), clone_params(src)
    oa = make[first](groups_of(a, lrs))
    ob = make[first](groups_of(b, lrs))
    start = {k: n(x).astype(np.float64) for k, x in src.items()}
    for step in range(10):
        grads = grads_for(src, 3, step)
        set_grads(a, grads)
        set_grads(b, grads)
        oa.step()
        ob.step()
    sd = ob.state_dict()
    c = clone_params({k: x.detach() for k, x in b.items()})
    oc = make[second](groups_of(c, lrs))
    oc.load_state_dict(sd)
    for p in c.values():
        st = oc.state[p]
        assert st["step"].device.type == "cpu" and st["step"].dtype == torch.float32
    for step in range(10, 20):
        grads = grads_for(src, 3, step)
        set_grads(a, grads)
        set_grads(c, grads)
        oa.step()
        oc.step()
    check_vs_torch(state_np(c, oc), state_np(a, oa), start)
    # and back: the second optimizer's state loads into the first kind
    od = make[first](groups_of(clone_params({k: x.detach() for k, x in c.items()}), lrs))
    od.load_state_dict(oc.state_dict())
    assert all(float(s["step"]) == 20 for s in od.state.values())


# ---------------------------------------------------------------- 4. controllers
def _controller_params(N, seed):
    rng = np.random.default_rng(seed)
    raw = {k: rng.normal(size=(N, w)).astype(np.float32) for k, w in WIDTHS.items()}
    raw["scales_raw"] = (raw["scales_raw"] * 0.5 - 3).astype(np.float32)
    raw["alphas_raw"] = rng.uniform(-8, 6, (N, 1)).astype(np.float32)
    raw["features"] = rng.normal(size=(N, 5)).astype(np.float32)
    return raw


def _run_controllers(opt_cls, raw, sd):
    params = {k: torch.nn.Parameter(t(v)) for k, v in raw.items()}
    groups = adam_groups(params) + [{"params": [params["features"]], "lr": 1e-2, "name": "features"}]
    opt = opt_cls(groups, lr=1e-3, eps=1e-15)
    if sd is not None:
        opt.load_state_dict(copy.deepcopy(sd))  # load_state_dict keeps the dict's CPU step tensors
    N = params["pws"].shape[0]
    g = torch.Generator(device=DEV).manual_seed(5)
    dens = DensityController(sense_size=2.0, verbose=False)
    dus = torch.randn((N, 2), device=DEV, generator=g) * 1e-5
    mask = torch.rand(N, device=DEV, generator=g) < 0.8
    dens.update_density_info(dus, mask)
    dens.update_gaussian_density(params, opt, generator=torch.Generator(device=DEV).manual_seed(6),
                                 extra=("features",))
    dens.reset_alpha(params, opt)
    mc = MCMCController(cap_max=int(params["pws"].shape[0] * 1.3), verbose=False)
    mc.relocate(params, opt, generator=torch.Generator(device=DEV).manual_seed(7), extra=("features",))
    mc.grow(params, opt, generator=torch.Generator(device=DEV).manual_seed(8), extra=("features",))
    mc.inject_noise(params, opt, generator=torch.Generator(device=DEV).manual_seed(9))
    gg = torch.Generator(device=DEV).manual_seed(10)
    for k, p in params.items():
        p.grad = torch.randn(p.shape, device=DEV, generator=gg)
    opt.step()
    return {k: (n(p).copy(), n(opt.state[p]["exp_avg"]).copy(), n(opt.state[p]["exp_avg_sq"]).copy(),
                float(opt.state[p]["step"])) for k, p in params.items()}, opt


def test_controllers_on_gaussian_adam_match_torch_adam():
    N = 20000
    raw = _controller_params(N, 3)
    # one real step gives both optimizers the same state
    params = {k: torch.nn.Parameter(t(v)) for k, v in raw.items()}
    groups = adam_groups(params) + [{"params": [params["features"]], "lr": 1e-2, "name": "features"}]
    seed_opt = torch.optim.Adam(groups, lr=1e-3, eps=1e-15)
    for p in params.values():
        p.grad = torch.randn_like(p)
    seed_opt.step()
    sd = seed_opt.state_dict()
    raw1 = {k: n(p).copy() for k, p in params.items()}
    raw1["alphas_raw"] = raw["alphas_raw"]
    ours, opt = _run_controllers(GaussianAdam, raw1, sd)
    ref, _ = _run_controllers(torch.optim.Adam, raw1, sd)
    assert isinstance(opt, GaussianAdam)
    assert ours.keys() == ref.keys() and ours["pws"][0].shape == ref["pws"][0].shape
    assert ours["pws"][0].shape[0] != N  # the controllers changed the row count
    check_vs_torch(ours, ref, {k: ref[k][0].astype(np.float64) for k in ref})  # 2 ulp(p) after one step


# ---------------------------------------------------------------- 5. the mask is safe
def _mask_scene(N, W, H, seed):
    from easygaussiansplatting_b200.scene import synthetic_scene
    sc = synthetic_scene(N, W, H, sh_dim=48, seed=seed)
    rng = np.random.default_rng(seed)
    pws = sc["pws"].copy()
    k = N // 10
    pws[:k, 2] = rng.uniform(-3.0, 0.19, k)                       # behind or too near the camera
    pws[k:2 * k, 0] += np.sign(rng.normal(size=k)) * 50.0 * pws[k:2 * k, 2]  # far off the frame
    sc["pws"] = pws.astype(np.float32)
    return sc


@pytest.mark.parametrize("kind", ["plain", "rgbd", "features"])
@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("filtered", [False, True])
def test_mask_covers_every_gradient(kind, aa, filtered):
    from easygaussiansplatting_b200.gsfunction import (Camera, GSFunctionFused, GSFunctionFusedFeatures,
                                                       GSFunctionFusedRGBD)
    N, W, H = 6000, 160, 96
    sc = _mask_scene(N, W, H, seed=40)
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]),
                 antialiased=aa)
    raw = dict(pws=sc["pws"], low_shs=sc["shs"][:, :3], high_shs=sc["shs"][:, 3:],
               alphas_raw=np.log(sc["alphas"] / (1 - sc["alphas"]))[:, None], scales_raw=np.log(sc["scales"]),
               rots_raw=sc["rots"])
    P = {k: torch.nn.Parameter(t(np.ascontiguousarray(v, np.float32))) for k, v in raw.items()}
    feats = torch.nn.Parameter(torch.randn((N, 5), device=DEV))
    alphas = torch.sigmoid(P["alphas_raw"])
    scales = torch.exp(P["scales_raw"])
    rots = torch.nn.functional.normalize(P["rots_raw"], dim=1)
    shs = torch.cat([P["low_shs"], P["high_shs"]], dim=1)
    us = torch.zeros((N, 2), device=DEV, requires_grad=True)
    f3 = (torch.rand(N, device=DEV) * 0.01) if filtered else None
    if kind == "plain":
        img, mask = GSFunctionFused.apply(P["pws"], shs, alphas, scales, rots, us, cam, f3)
        loss = (img ** 2).sum()
    elif kind == "rgbd":
        img, dep, alp, mask = GSFunctionFusedRGBD.apply(P["pws"], shs, alphas, scales, rots, us, cam, f3)
        loss = (img ** 2).sum() + (dep * 0.1).sum() + alp.sum()
    else:
        img, fmap, mask = GSFunctionFusedFeatures.apply(P["pws"], shs, alphas, scales, rots, us, feats, cam, f3)
        loss = (img ** 2).sum() + (fmap ** 2).sum()
    loss.backward()
    m = n(mask).astype(bool)
    assert m.shape == (N,) and 0 < m.sum() < N - N // 10
    touched = np.zeros(N, bool)
    tensors = list(P.values()) + ([feats] if kind == "features" else [])
    for p in tensors:
        touched |= (n(p.grad).reshape(N, -1) != 0).any(axis=1)
    assert touched.sum() > N // 4
    assert not (touched & ~m).any(), int((touched & ~m).sum())


# ---------------------------------------------------------------- 6. training
def _train(opt_kind, selective, steps=60):
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused
    from easygaussiansplatting_b200.scene import synthetic_scene
    W, H, N = 160, 120, 4000
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=50)
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]))
    us0 = torch.zeros((N, 2), device=DEV)
    with torch.no_grad():
        target, _ = GSFunctionFused.apply(t(sc["pws"]), t(sc["shs"]), t(sc["alphas"][:, None]), t(sc["scales"]),
                                          t(sc["rots"]), us0, cam)
    rng = np.random.default_rng(51)
    raw = dict(pws=sc["pws"] + rng.normal(size=(N, 3)).astype(np.float32) * 0.02, low_shs=np.zeros((N, 3)),
               high_shs=np.zeros((N, 45)), alphas_raw=np.zeros((N, 1)), scales_raw=np.log(sc["scales"]) - 0.2,
               rots_raw=sc["rots"])
    params = {k: torch.nn.Parameter(t(np.ascontiguousarray(v, np.float32))) for k, v in raw.items()}
    groups = adam_groups(params)
    for g in groups:
        g["lr"] = dict(pws=1.6e-4, low_shs=0.02).get(g["name"], g["lr"])
    opt = (GaussianAdam if opt_kind == "ours" else torch.optim.Adam)(groups, lr=1e-3, eps=1e-15)
    losses = []
    for _ in range(steps):
        P = params
        shs = torch.cat([P["low_shs"], P["high_shs"][:, :9]], dim=1)
        us = torch.zeros((N, 2), device=DEV, requires_grad=True)
        img, mask = GSFunctionFused.apply(P["pws"], shs, torch.sigmoid(P["alphas_raw"]), torch.exp(P["scales_raw"]),
                                          torch.nn.functional.normalize(P["rots_raw"], dim=1), us, cam)
        loss = (img - target).abs().mean()
        opt.zero_grad()
        loss.backward()
        if selective:
            opt.step(visibility=mask)
        else:
            opt.step()
        losses.append(float(loss.detach()))
    return np.array(losses)


def test_training_dense_tracks_torch_adam():
    ours = _train("ours", False)
    ref = _train("torch", False)
    # the same fp32 operations on the same gradients: what differs comes from the rasterizer
    # backward's float atomics, which make neither run bit-reproducible
    assert np.abs(ours - ref).max() <= 1e-2 * ref[0], np.abs(ours - ref).max()
    assert ours[-5:].mean() < 0.6 * ours[:5].mean()


def test_training_selective_reduces_the_loss():
    losses = _train("ours", True)
    assert np.isfinite(losses).all()
    assert losses[-5:].mean() < 0.6 * losses[:5].mean(), losses[::10]
