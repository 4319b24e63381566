"""2D Gaussian Splatting on the GPU: the four planes and every gradient against the fp64 oracle
(oracle/surfel_oracle.py, binned on the kernels' own us / depths / areas), the capacity path against
the exact one, the fronto-parallel identities, GSFunctionSurfel through autograd and its refusals."""
import numpy as np
import pytest
import torch

from oracle import surfel_oracle as so

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def scene(N, W, H, k=16, seed=0, z=(2.0, 6.0), spread=1.0):
    rng = np.random.default_rng(seed)
    fx = fy = 0.8 * W
    cx, cy = W / 2 - 0.3, H / 2 + 0.2
    zz = rng.uniform(*z, N)
    pws = np.stack([rng.uniform(-spread, spread, N) * zz * W / (2 * fx), rng.uniform(-spread, spread, N) * zz * H / (2 * fy),
                    zz], 1)
    rots = rng.normal(size=(N, 4))
    scales = np.stack([rng.uniform(0.02, 0.15, N), rng.uniform(0.02, 0.15, N), rng.uniform(0.0, 0.05, N)], 1)
    shs = rng.normal(scale=0.3, size=(N, 3 * k))
    alphas = rng.uniform(0.05, 0.95, N)
    f = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    return dict(pws=f(pws), rots=f(rots), scales=f(scales), shs=f(shs), alphas=f(alphas), Rcw=f(np.eye(3)),
                tcw=f(np.zeros(3)), twc=f(np.zeros(3)), fx=fx, fy=fy, cx=cx, cy=cy, W=W, H=H)


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def gpu_frame(sc, dl=None, capacity=False):
    from easygaussiansplatting_b200 import ops
    P = {k: T(sc[k]) for k in ("pws", "rots", "scales", "shs", "alphas", "Rcw", "tcw", "twc")}
    cam = (sc["fx"], sc["fy"], sc["cx"], sc["cy"], sc["W"], sc["H"])
    us, depths, areas, colors, recs = ops.surfel_preprocess(P["pws"], P["rots"], P["scales"], P["shs"], P["alphas"],
                                                            P["Rcw"], P["tcw"], P["twc"], *cam)
    pre = dict(us=us.cpu().numpy(), depths=depths.cpu().numpy().copy(), areas=areas.cpu().numpy().copy())
    out = ops.splat_surfel(sc["H"], sc["W"], us, depths, areas, recs, capacity=capacity)
    res = dict(pre=pre, out=[o.cpu().numpy() for o in out])
    if dl is not None:
        rows = ops.splatB_surfel(sc["H"], sc["W"], recs, out[1], out[2], out[3], out[4], *[T(d) for d in dl])
        g = ops.surfel_preprocessB(P["pws"], P["rots"], P["scales"], P["shs"], P["Rcw"], P["tcw"], P["twc"], *cam, rows)
        res["grads"] = dict(zip(("pws", "shs", "alphas", "scales", "rots", "us"), [t.cpu().numpy() for t in g]))
        res["rows"] = rows.cpu().numpy()
    torch.cuda.synchronize()
    return res


def oracle_frame(sc, gpu_pre, dl):
    pre = so.preprocess(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                        sc["fy"], sc["cx"], sc["cy"])
    bins = so.orc.bin(sc["H"], sc["W"], gpu_pre["us"], gpu_pre["depths"].copy(), gpu_pre["areas"].copy())
    fwd = so.render(sc["H"], sc["W"], pre, sc["alphas"], bins)
    rows = so.render_backward(sc["H"], sc["W"], pre, sc["alphas"], bins, fwd, *dl)
    return pre, fwd, so.preprocess_backward(pre, rows)


def upstream(H, W, seed=1):
    rng = np.random.default_rng(seed)
    return [rng.normal(size=s).astype(np.float32) for s in ((3, H, W), (H, W), (H, W), (3, H, W))]


@pytest.mark.parametrize("N,W,H,k,spread", [(3, 40, 24, 1, 0.3), (60, 72, 40, 4, 1.1), (400, 90, 60, 16, 1.2),
                                             (1500, 64, 48, 9, 1.0), (20000, 160, 96, 16, 1.0)])
def test_planes_and_gradients_match_oracle(N, W, H, k, spread):
    sc = scene(N, W, H, k=k, seed=N, spread=spread)
    # the oracle's ambiguous pixels (a threshold within its margin) get no upstream gradient: a pixel's
    # terms are all proportional to its own dL/dplanes, so every gradient is then compared exactly
    g0 = gpu_frame(sc)
    pre, fwd, _ = oracle_frame(sc, g0["pre"], upstream(H, W))
    amb = fwd["ambiguous"]
    assert (~amb).mean() > 0.95
    dl = [np.where(amb, 0.0, d).astype(np.float32) for d in upstream(H, W)]
    g = gpu_frame(sc, dl)
    _, _, ref = oracle_frame(sc, g["pre"], dl)
    ok = ~amb
    image, contrib, ftau, ranges, _, depth, alpha, normal = g["out"]
    for name, got, want in (("image", image, fwd["image"]), ("normal", normal, fwd["normal"])):
        assert np.abs(got - want).max(axis=0)[ok].max() < 1e-4, name
    assert np.abs(alpha - fwd["alpha"])[ok].max() < 1e-4
    assert np.abs(depth - fwd["depth"])[ok].max() < 1e-4 * max(1.0, np.abs(fwd["depth"]).max())
    assert (contrib == fwd["contrib"])[ok].all()
    lens = ranges[:, 1] - ranges[:, 0]
    if N >= 1500:  # dense tiles: per-block entries and a multi-chunk ring walk in both directions
        assert lens.max() > 96 and (contrib > 64).any()
    if N == 60:
        assert 0 < lens.max() <= 32  # whole-tile entries only
    for name in ("pws", "shs", "alphas", "scales", "rots", "us"):
        want = ref[name].reshape(g["grads"][name].shape)
        err = np.abs(g["grads"][name] - want).max() / max(np.abs(want).max(), 1e-12)
        assert err < 1e-4, (name, err)
    assert (g["grads"]["scales"][:, 2] == 0).all()


def test_empty_scene_and_culled_surfels():
    sc = scene(0, 33, 17)
    g = gpu_frame(sc, upstream(17, 33))
    assert all(np.all(o == 0) for o in (g["out"][0], g["out"][5], g["out"][6], g["out"][7]))
    assert g["grads"]["pws"].shape == (0, 3)
    # surfels at the z = 0.2 cull and across the image border
    sc = scene(40, 50, 30, k=1, seed=5, z=(0.19, 0.21), spread=1.6)
    g = gpu_frame(sc, upstream(30, 50))
    pre, fwd, ref = oracle_frame(sc, g["pre"], upstream(30, 50))
    culled = sc["pws"][:, 2] < np.float32(0.2)
    assert culled.any() and (~culled).any()
    assert (g["pre"]["depths"][culled] == -1).all()
    ok = ~fwd["ambiguous"]
    assert np.abs(g["out"][0] - fwd["image"]).max(axis=0)[ok].max() < 1e-4
    assert (g["grads"]["pws"][culled] == 0).all() and (g["grads"]["rots"][culled] == 0).all()


def test_fronto_parallel_identities():
    rng = np.random.default_rng(4)
    N, z0, W, H = 300, 3.0, 70, 45
    sc = scene(N, W, H, k=1, seed=4)
    ang = rng.uniform(0, np.pi, N)
    sc["rots"] = np.stack([np.cos(ang / 2), np.zeros(N), np.zeros(N), np.sin(ang / 2)], 1).astype(np.float32)
    sc["pws"][:, 2] = z0
    g = gpu_frame(sc)
    _, _, _, _, _, depth, alpha, normal = g["out"]
    assert alpha.max() > 0.5
    np.testing.assert_allclose(depth, z0 * alpha, atol=2e-5)
    np.testing.assert_allclose(normal[2], -alpha, atol=1e-6)
    assert np.abs(normal[:2]).max() == 0


def test_capacity_path_matches_exact_path():
    from easygaussiansplatting_b200 import ops
    sc = scene(20000, 160, 96, k=16, seed=7)
    dl = upstream(96, 160)
    exact = gpu_frame(sc, dl)
    stats = dict(ops.CAPACITY_STATS)
    first = gpu_frame(sc, dl, capacity=True)   # exact, learns the bounds
    second = gpu_frame(sc, dl, capacity=True)  # capacity path
    assert ops.CAPACITY_STATS["capacity_frames"] > stats["capacity_frames"]
    for a, b, c in zip(exact["out"], first["out"], second["out"]):
        assert np.array_equal(a, b) and np.array_equal(a, c)
    # (the gradient rows are sums of float atomics: equal up to their order)
    for k in exact["grads"]:
        a, b = exact["grads"][k], second["grads"][k]
        assert np.abs(a - b).max() <= 1e-5 * np.abs(a).max(), k
    # an outgrown frame: the same shape with four times the patches falls back to the exact path
    big = dict(sc)
    big["scales"] = (sc["scales"] * 2.5).astype(np.float32)
    outgrown = ops.CAPACITY_STATS["outgrown"]
    got = gpu_frame(big, None, capacity=True)
    ref = gpu_frame(big, None)
    assert ops.CAPACITY_STATS["outgrown"] == outgrown + 1
    for a, b in zip(got["out"], ref["out"]):
        assert np.array_equal(a, b)


def test_gsfunction_surfel_autograd_refusals_and_skipped_planes():
    from easygaussiansplatting_b200 import _lib
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionSurfel
    sc = scene(200, 64, 40, k=4, seed=11)
    cam = Camera(64, 40, sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(sc["Rcw"]), T(sc["tcw"]), T(sc["twc"]))
    P = {k: T(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    al = T(sc["alphas"][:, None]).requires_grad_()
    us = torch.zeros((200, 2), device=DEV, requires_grad=True)
    image, depth, alpha, normal, mask = GSFunctionSurfel.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us, cam)
    dl = upstream(40, 64)
    loss = sum((p * T(d)).sum() for p, d in zip((image, depth, alpha, normal), dl))
    loss.backward()
    g = gpu_frame(sc, dl)
    assert np.array_equal(image.detach().cpu().numpy(), g["out"][0])
    for name, t in (("pws", P["pws"]), ("shs", P["shs"]), ("scales", P["scales"]), ("rots", P["rots"]), ("us", us)):
        np.testing.assert_allclose(t.grad.cpu().numpy(), g["grads"][name], rtol=0, atol=1e-6 * np.abs(g["grads"][name]).max())
    np.testing.assert_allclose(al.grad.cpu().numpy()[:, 0], g["grads"]["alphas"], atol=1e-6)
    assert mask.dtype == torch.bool
    # a frame whose loss reads no plane the backward can use launches no backward rasterizer
    lib = _lib.load()
    kid = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())].index("draw_surfel_backward")
    n0 = lib.gsb_profile_launches(kid)
    out = GSFunctionSurfel.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us, cam)
    (out[2].sum() * 0).backward()
    n1 = lib.gsb_profile_launches(kid)
    assert n1 == n0 + 1
    from easygaussiansplatting_b200 import ops
    pre = ops.surfel_preprocess(P["pws"].detach(), P["rots"].detach(), P["scales"].detach(), P["shs"].detach(),
                                al.detach().reshape(-1), cam.Rcw, cam.tcw, cam.twc, cam.fx, cam.fy, cam.cx, cam.cy,
                                64, 40)
    recs = pre[4]
    img, con, tau, rng_, gs, *_ = ops.splat_surfel(40, 64, pre[0], pre[1], pre[2], recs)
    rows = ops.splatB_surfel(40, 64, recs, con, tau, rng_, gs)
    torch.cuda.synchronize()
    assert lib.gsb_profile_launches(kid) == n1 and (rows == 0).all()
    # refused options
    for kw in (dict(antialiased=True), dict(camera_model="ortho")):
        c = Camera(64, 40, sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(sc["Rcw"]), T(sc["tcw"]), T(sc["twc"]), **kw)
        with pytest.raises(ValueError):
            GSFunctionSurfel.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us, c)
    with pytest.raises(ValueError):
        GSFunctionSurfel.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us, cam, torch.zeros(200, device=DEV))
    with pytest.raises(ValueError):
        GSFunctionSurfel.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us, cam, None, torch.zeros_like(us))
    cam.grad_exchange = object()
    with pytest.raises(ValueError):
        GSFunctionSurfel.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us, cam)


def test_short_training_lowers_the_loss():
    """surfels fitted to a target rendered from other surfels: Adam on all parameters, 60 steps"""
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionSurfel
    W, H = 64, 48
    tgt = scene(300, W, H, k=1, seed=21)
    cam = Camera(W, H, tgt["fx"], tgt["fy"], tgt["cx"], tgt["cy"], T(tgt["Rcw"]), T(tgt["tcw"]), T(tgt["twc"]))
    with torch.no_grad():
        ref = GSFunctionSurfel.apply(T(tgt["pws"]), T(tgt["shs"]), T(tgt["alphas"][:, None]), T(tgt["scales"]),
                                     T(tgt["rots"]), torch.zeros((300, 2), device=DEV), cam)
    sc = scene(300, W, H, k=1, seed=22)
    P = [T(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")]
    araw = T(np.log(sc["alphas"] / (1 - sc["alphas"]))[:, None]).requires_grad_()
    opt = torch.optim.Adam(P + [araw], lr=5e-3)
    losses = []
    for _ in range(60):
        us = torch.zeros((300, 2), device=DEV, requires_grad=True)
        img, depth, alpha, normal, _ = GSFunctionSurfel.apply(P[0], P[1], torch.sigmoid(araw), P[2].abs(), P[3], us, cam)
        loss = (img - ref[0]).abs().mean() + 0.1 * (alpha - ref[2]).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert np.isfinite(losses).all()
    assert losses[-1] < 0.7 * losses[0]


def _surfel_training_setup(N, W, H, seed):
    """a target rendered from one surfel scene, and the raw training tensors of a perturbed half of it"""
    from easygaussiansplatting_b200.gau_io import adam_groups
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionSurfel
    from easygaussiansplatting_b200.scene import synthetic_scene
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=seed)
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(sc["Rcw"]), T(sc["tcw"]), T(sc["twc"]))
    with torch.no_grad():
        target = GSFunctionSurfel.apply(T(sc["pws"]), T(sc["shs"]), T(sc["alphas"][:, None]), T(sc["scales"]),
                                        T(sc["rots"]), torch.zeros((N, 2), device=DEV), cam)
    N0 = N // 2
    rng = np.random.default_rng(seed + 1)
    a0 = np.log(sc["alphas"][:N0] / (1 - sc["alphas"][:N0])).astype(np.float32)
    a0[rng.random(N0) < 0.1] = -8.0  # nearly transparent: pruned / relocated
    s_raw = np.log(sc["scales"][:N0]).astype(np.float32)
    s_raw[:, 2] = np.log(1e-3)  # the third scale is not rendered: kept small for the splits
    raw = dict(pws=sc["pws"][:N0] + rng.normal(size=(N0, 3)).astype(np.float32) * 0.02,
               low_shs=np.zeros((N0, 3), np.float32), high_shs=np.zeros((N0, 45), np.float32),
               alphas_raw=a0.reshape(N0, 1), scales_raw=s_raw, rots_raw=sc["rots"][:N0])
    params = {k: torch.nn.Parameter(T(np.ascontiguousarray(v, dtype=np.float32))) for k, v in raw.items()}
    groups = adam_groups(params)
    for g in groups:
        g["lr"] = dict(pws=1.6e-4, low_shs=0.02).get(g["name"], g["lr"])
    return cam, target, params, groups


def _surfel_step(params, cam, target):
    from easygaussiansplatting_b200.gsfunction import GSFunctionSurfel
    P = params
    alphas = torch.sigmoid(P["alphas_raw"])
    scales = torch.exp(P["scales_raw"])
    rots = torch.nn.functional.normalize(P["rots_raw"], dim=1)
    shs = torch.cat([P["low_shs"], P["high_shs"][:, :9]], dim=1)
    us = torch.zeros((P["pws"].shape[0], 2), device=DEV, requires_grad=True)
    img, depth, alpha, normal, mask = GSFunctionSurfel.apply(P["pws"], shs, alphas, scales, rots, us, cam)
    loss = (img - target[0]).abs().mean() + 0.1 * (alpha - target[2]).abs().mean()
    loss.backward()
    return float(loss.detach()), us, mask


def test_training_with_density_control_and_gaussian_adam():
    """surfels densified by DensityController on us.grad (the screen-space shift statistic, the
    reference's threshold) and stepped by GaussianAdam: prunes, clones and splits happen, the loss falls"""
    from easygaussiansplatting_b200.density import DensityController
    from easygaussiansplatting_b200.optim import GaussianAdam
    cam, target, params, groups = _surfel_training_setup(6000, 160, 120, 40)
    opt = GaussianAdam(groups, lr=1e-3)
    ctl = DensityController(sense_size=5.0, verbose=False)
    N0 = params["pws"].shape[0]
    losses, changed = [], False
    for step in range(90):
        opt.zero_grad()
        loss, us, mask = _surfel_step(params, cam, target)
        ctl.update_density_info(us.grad, mask)
        opt.step()
        losses.append(loss)
        if step in (29, 59):
            before = params["pws"].shape[0]
            ctl.update_gaussian_density(params, opt)
            assert params["pws"].shape[0] != before
            changed = True
        assert all(torch.isfinite(p).all() for p in params.values())
    assert changed and params["pws"].shape[0] > 0.95 * N0  # the pruned tenth came back through clones / splits
    assert np.mean(losses[-5:]) < 0.7 * np.mean(losses[:5]), losses[::10]


def test_training_with_mcmc():
    """surfels relocated, grown to the cap and noised by MCMCController: the loss falls"""
    from easygaussiansplatting_b200.density import MCMCController
    cam, target, params, groups = _surfel_training_setup(6000, 160, 120, 50)
    opt = torch.optim.Adam(groups, lr=1e-3)
    cap = 4000
    ctl = MCMCController(cap, grow_rate=0.1, noise_lr=1e3, verbose=False)
    rng = torch.Generator(device=DEV).manual_seed(51)
    losses = []
    for step in range(80):
        opt.zero_grad()
        loss, _, _ = _surfel_step(params, cam, target)
        opt.step()
        ctl.inject_noise(params, opt, generator=rng)
        losses.append(loss)
        if step % 10 == 9:
            ctl.relocate(params, opt, generator=rng)
            ctl.grow(params, opt, generator=rng)
        assert params["pws"].shape[0] <= cap
        assert all(torch.isfinite(p).all() for p in params.values())
    assert params["pws"].shape[0] == cap
    assert np.mean(losses[-5:]) < 0.7 * np.mean(losses[:5]), losses[::10]
