"""The OpenCV radial-tangential camera model on the H100: ops.preprocess / preprocessB against the fp64
oracle (oracle/opencv_oracle.py) at every SH degree with and without antialiasing, depth and the camera
gradient, for zero, SIMPLE_RADIAL-like, COLMAP-like and strong-barrel coefficients; the validity cull;
zero coefficients against the pinhole entry points; whole steps of the fused classes against
opencv_oracle.step; the graphed and multi-view steps against the eager class; a config-2-sized frame;
and a short training run."""
import numpy as np
import pytest
import torch

from easygaussiansplatting_b200 import ops
from easygaussiansplatting_b200.gsfunction import (Camera, GSFunctionFused, GSFunctionFusedFeatures,
                                                   GSFunctionFusedPose, GSFunctionFusedRGBD,
                                                   GSFunctionFusedRGBDPose)
from easygaussiansplatting_b200.scene import COLMAP_LIKE_OPENCV, camera_model_scene, upstream_gradient
from oracle import opencv_oracle as ocv
from oracle import oracle as orc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ZERO = (0.0, 0.0, 0.0, 0.0)
SIMPLE_RADIAL = (0.08, 0.0, 0.0, 0.0)
COLMAP = COLMAP_LIKE_OPENCV[0] + COLMAP_LIKE_OPENCV[1]
BARREL = (-0.45, 0.05, 0.0, 0.0)  # folds inside the frame's corners
KSETS = [ZERO, SIMPLE_RADIAL, COLMAP, BARREL]
KIDS = ["zero", "simple_radial", "colmap", "barrel"]
oaa = ocv.oaa


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _kw(k):
    return dict(camera_model="opencv", radial_coeffs=tuple(k[:2]), tangential_coeffs=tuple(k[2:]))


def _scene(k, N, W, H, k3, seed):
    sc = camera_model_scene(N, W, H, "opencv", k[:2], sh_dim=3 * k3, seed=seed, tangential_coeffs=k[2:])
    a, b = 0.1, -0.05
    Ry = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    Rx = np.array([[1, 0, 0], [0, np.cos(b), -np.sin(b)], [0, np.sin(b), np.cos(b)]])
    R, t = Ry @ Rx, np.array([0.1, -0.05, 0.2])
    sc["pws"] = np.ascontiguousarray((sc["pws"].astype(np.float64) - t) @ R, np.float32)
    sc["Rcw"], sc["tcw"], sc["twc"] = R.astype(np.float32), t.astype(np.float32), (-(R.T @ t)).astype(np.float32)
    return sc


def _args(sc):
    return (T(sc["pws"]), T(sc["rots"]), T(sc["scales"]), T(sc["shs"]), T(sc["Rcw"]), T(sc["tcw"]), T(sc["twc"]),
            sc["fx"], sc["fy"], sc["cx"], sc["cy"], sc["width"], sc["height"])


def _stages(sc, k):
    return ocv.stages(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                      sc["fy"], sc["cx"], sc["cy"], sc["width"], sc["height"], model="opencv", k=k)


def _pc(sc):
    return sc["pws"].astype(np.float64) @ sc["Rcw"].astype(np.float64).T + sc["tcw"]


def _band(sc, k):
    """rows within 1e-5 of the near plane, or 1e-4 of the opencv cull or clamp"""
    pc = _pc(sc)
    band = np.abs(pc[:, 2] - 0.2) < 1e-5
    return band | ((pc[:, 2] > 0.2) & ocv.opencv_band(pc, k, sc["fx"], sc["fy"], sc["cx"], sc["cy"], sc["width"],
                                                      sc["height"]))


def _close(got, ref, rows, tol=1e-4, what=""):
    got = np.asarray(got, np.float64).reshape(len(rows), -1)[rows]
    ref = np.asarray(ref, np.float64).reshape(len(rows), -1)[rows]
    if ref.size == 0:
        return
    err = np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30)
    assert err < tol, "%s: %.3g of max|ref|" % (what, err)


def _moment_grads(m, ci):
    """dL/du, dL/dconic, dL/dcolour, dL/dalpha of moment rows m against the forward's conics ci"""
    cig = ci.astype(np.float64)
    none = (m[:, 0] == 0) & (m[:, 1] == 0)
    gu = np.where(none[:, None], 0.0, -np.stack([cig[:, 0] * m[:, 0] + cig[:, 1] * m[:, 1],
                                                 cig[:, 1] * m[:, 0] + cig[:, 2] * m[:, 1]], 1))
    gci = np.stack([-0.5 * m[:, 2], -m[:, 3], -0.5 * m[:, 4]], 1).astype(np.float64)
    return gu, gci, m[:, 6:9].astype(np.float64), m[:, 5].astype(np.float64)


def _per_gaussian(sc, k, aa, depth, pose, seed=0, pose_only=False):
    """preprocess + preprocessB with random moment rows, against the oracle chain"""
    N = len(sc["pws"])
    args = _args(sc)
    al = T(sc["alphas"])
    pre = ops.preprocess(*args, alphas=al, antialiased=aa, **_kw(k))
    us, ci, col, dep, ar = (x.cpu().numpy() for x in pre[:5])
    st = _stages(sc, k)
    keep = st["keep"]
    thin = oaa.thin(sc["scales"])
    sure = ~_band(sc, k)
    assert np.array_equal((dep >= 0.2)[sure], keep[sure])
    ok = keep & sure & ~thin
    _close(us, st["us"], ok, what="us")
    _close(ci, st["ci"], ok, what="conic")
    _close(col, st["col"], np.ones(N, bool), what="colour")
    s = oaa.scale(st["c2"], keep)
    if aa:
        ok &= ~oaa.flagged(sc["scales"], s)
        np.testing.assert_allclose(pre[6].cpu().numpy()[ok], (s["rho"] * sc["alphas"])[ok], rtol=1e-3)
    rng = np.random.default_rng(seed)
    m = rng.normal(size=(N, 9)).astype(np.float32)
    m[rng.random(N) < 0.1] = 0.0
    gz = rng.normal(size=N).astype(np.float32) if depth else None
    out = ops.preprocessB(*args, None, None, None, moments=T(m), cinv2ds=pre[1], dloss_ddepths=T(gz) if depth else None,
                          camera_grad=pose, pose_only=pose_only, antialiased=aa, alphas=al if aa else None, **_kw(k))
    torch.cuda.synchronize()
    gu, gci, gcol, ga = _moment_grads(m, ci)
    Rcw = sc["Rcw"]
    ch = orc.chain_backward(Rcw, gu.reshape(N, 1, 2), gci.reshape(N, 1, 3), ga.reshape(N, 1, 1),
                            gcol.reshape(N, 1, 3), *st["J"])
    ref = {n: ch[n] for n in ("pws", "scales", "rots", "shs")}
    if depth:
        ref["pws"] = ref["pws"] + ocv.ordb.chain_depth(Rcw, gz.reshape(N, 1, 1), st["depths"])
    dal = ga
    W, H = sc["width"], sc["height"]
    per = ocv.camera_grad(st, sc["pws"], Rcw, sc["fx"], sc["fy"], W, H, gu, gci, gcol, gz, model="opencv")["per"]
    if aa:
        gc2 = oaa.dcov2d_addend(st["c2"], keep, sc["alphas"], ga)
        add = oaa.chain(st, Rcw, gc2)
        for n in ("pws", "scales", "rots"):
            ref[n] = ref[n] + add[n]
        dal = s["rho"] * ga
        per = per + ocv.camera_grad(oaa._identity_conic(st), sc["pws"], Rcw, sc["fx"], sc["fy"], W, H,
                                    np.zeros((N, 2)), gc2, np.zeros((N, 3)), model="opencv")["per"]
    rows = sure & ~thin
    if aa:
        rows &= ~oaa.flagged(sc["scales"], s)
    if not pose_only:
        gpw, gsh, gs, gq, dus, dalk = (x.cpu().numpy() for x in out[:6])
        for n, got in (("pws", gpw), ("scales", gs), ("rots", gq), ("shs", gsh)):
            _close(got, ref[n], rows, what="d" + n)
        _close(dus, gu, rows, tol=1e-5, what="dus")
        _close(dalk, dal, rows, tol=1e-5, what="dalphas")
    if pose:
        g = torch.cat([x.reshape(-1) for x in out[-1]]).cpu().numpy()
        per_ok = np.where(rows[:, None], per, 0.0)
        g_ref = per.sum(0)
        err = np.abs(g - g_ref) / np.maximum(np.abs(per).sum(0), 1e-30)
        assert err.max() < 1e-4, err.max()
        assert np.abs(per_ok.sum(0)).max() > 0
    return out


@pytest.mark.parametrize("k", KSETS, ids=KIDS)
@pytest.mark.parametrize("k3", [1, 4, 9, 16])
@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("depth,pose", [(False, False), (True, False), (False, True), (True, True)])
def test_preprocess_against_oracle(k, k3, aa, depth, pose):
    sc = _scene(k, 1037, 320, 240, k3, seed=k3)
    _per_gaussian(sc, k, aa, depth, pose, seed=k3 + 7 * aa)


@pytest.mark.parametrize("k", KSETS, ids=KIDS)
@pytest.mark.parametrize("aa", [False, True])
def test_pose_only_against_oracle(k, aa):
    sc = _scene(k, 777, 320, 240, 4, seed=3)
    out = _per_gaussian(sc, k, aa, True, True, pose_only=True)
    assert out[0] is None


@pytest.mark.parametrize("k", KSETS, ids=KIDS)
def test_empty_and_unaligned(k):
    sc = _scene(k, 0, 64, 48, 4, seed=1)
    pre = ops.preprocess(*_args(sc), alphas=T(sc["alphas"]), **_kw(k))
    assert pre[0].shape == (0, 2)
    out = ops.preprocessB(*_args(sc), None, None, None, moments=torch.zeros((0, 9), device=DEV), cinv2ds=pre[1],
                          camera_grad=True, **_kw(k))
    assert out[0].shape == (0, 3) and float(torch.cat([x.reshape(-1) for x in out[-1]]).abs().sum()) == 0.0
    sc = _scene(k, 129, 64, 48, 4, seed=2)
    _per_gaussian(sc, k, True, True, True, seed=5)
    base = ops.preprocess(*_args(sc), alphas=T(sc["alphas"]), **_kw(k))
    rots = torch.empty((129 * 4 + 1,), device=DEV)[1:].view(129, 4)
    rots.copy_(T(sc["rots"]))
    a = list(_args(sc)); a[1] = rots
    odd = ops.preprocess(*a, alphas=T(sc["alphas"]), **_kw(k))
    for x, y in zip(base, odd):
        assert torch.equal(x, y)


@pytest.mark.parametrize("k,which", [(BARREL, "rho"), ((0.0, 0.0, 0.2, 0.0), "det")])
def test_validity_cull(k, which):
    """rows beyond rho_valid (BARREL) and where det Ddelta <= 0 (a strong tangential term) are culled like
    z < 0.2: depth -1, zero area, zero geometry gradient"""
    sc = _scene(k, 3000, 320, 240, 1, seed=4)
    pre = ops.preprocess(*_args(sc), alphas=T(sc["alphas"]), **_kw(k))
    dep, ar = pre[3].cpu().numpy(), pre[4].cpu().numpy()
    pc = _pc(sc)
    valid, drho, det = ocv.opencv_valid(pc, k)
    folded = (pc[:, 2] >= 0.2) & ~valid & ~_band(sc, k)
    assert folded.sum() > 20
    assert ((drho < 0) if which == "rho" else (det < 0))[folded].sum() > 20
    assert (dep[folded] == -1).all() and (ar[folded] == 0).all()
    _per_gaussian(sc, k, True, True, True)
    m = torch.ones((3000, 9), device=DEV)
    g = ops.preprocessB(*_args(sc), None, None, None, moments=m, cinv2ds=pre[1], **_kw(k))
    fm = torch.from_numpy(folded).to(DEV)
    assert float(g[2][fm].abs().max()) == 0.0 and float(g[3][fm].abs().max()) == 0.0


@pytest.mark.parametrize("k3", [1, 16])
@pytest.mark.parametrize("aa", [False, True])
def test_zero_coefficients_against_the_pinhole_entry_points(k3, aa):
    """the forward outputs to fp32 rounding everywhere; the gradients on rows the clamp does not touch
    (pinhole keeps the reference's unclamped-x, y derivative of the clamped J)"""
    sc = _scene(ZERO, 2000, 320, 240, k3, seed=k3)
    sc["pws"][::17, 0] *= 3.0  # beyond the clamp
    sc["pws"][::23, 2] = -1.0  # culled
    args = _args(sc)
    al = T(sc["alphas"])
    N = len(sc["pws"])
    ref = ops.preprocess(*args, alphas=al, antialiased=aa)
    got = ops.preprocess(*args, alphas=al, antialiased=aa, **_kw(ZERO))
    torch.cuda.synchronize()
    assert torch.equal(ref[3], got[3]) and torch.equal(ref[2], got[2])
    keep = ref[3].cpu().numpy() >= 0.2
    for i, what in ((0, "us"), (1, "conic")):
        _close(got[i].cpu().numpy(), ref[i].cpu().numpy(), keep, tol=1e-5, what=what)
    dar = (got[4] - ref[4]).abs().cpu().numpy()
    assert dar.max() <= 1 and (dar > 0).mean() < 0.01
    if aa:
        _close(got[6].cpu().numpy(), ref[6].cpu().numpy(), np.ones(N, bool), tol=1e-5, what="alphas_eff")
    pc = _pc(sc)
    lx, ly = 1.3 * sc["width"] / (2 * sc["fx"]), 1.3 * sc["height"] / (2 * sc["fy"])
    unc = keep & (np.abs(pc[:, 0] / pc[:, 2]) < lx * (1 - 1e-4)) & (np.abs(pc[:, 1] / pc[:, 2]) < ly * (1 - 1e-4))
    assert (keep & ~unc).sum() > 50
    m = T(np.random.default_rng(k3).normal(size=(N, 9)).astype(np.float32))
    gz = T(np.random.default_rng(k3 + 1).normal(size=N).astype(np.float32))
    r = ops.preprocessB(*args, None, None, None, moments=m, cinv2ds=ref[1], dloss_ddepths=gz, antialiased=aa,
                        alphas=al if aa else None)
    o = ops.preprocessB(*args, None, None, None, moments=m, cinv2ds=ref[1], dloss_ddepths=gz, antialiased=aa,
                        alphas=al if aa else None, **_kw(ZERO))
    torch.cuda.synchronize()
    rows = unc & ~oaa.thin(sc["scales"])
    for i, what in enumerate(("dpws", "dshs", "dscales", "drots", "dus", "dalphas")):
        _close(o[i].cpu().numpy(), r[i].cpu().numpy(), rows, tol=1e-4, what=what)


def _cam(sc, k, aa=False):
    return Camera(sc["width"], sc["height"], sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(sc["Rcw"]), T(sc["tcw"]),
                  T(sc["twc"]), antialiased=aa, **_kw(k))


def _params(sc):
    P = {n: T(sc[n]).requires_grad_() for n in ("pws", "shs", "scales", "rots")}
    P["alphas"] = T(sc["alphas"][:, None]).requires_grad_()
    P["us"] = torch.zeros((len(sc["pws"]), 2), device=DEV, requires_grad=True)
    return P


@pytest.mark.parametrize("k", [COLMAP, BARREL], ids=["colmap", "barrel"])
@pytest.mark.parametrize("cls", ["fused", "rgbd", "pose", "rgbdpose", "features"])
@pytest.mark.parametrize("aa,filt", [(False, False), (True, False), (False, True), (True, True)])
def test_whole_step_against_oracle(k, cls, aa, filt):
    W, H, N = 96, 64, 600
    sc = _scene(k, N, W, H, 4, seed=5)
    cam = _cam(sc, k, aa)
    P = _params(sc)
    f3 = None
    if filt:
        f3 = np.random.default_rng(1).uniform(0.0, 0.3, N).astype(np.float32) * sc["scales"].min(1)
    ft = T(f3) if filt else None
    rgbd = cls in ("rgbd", "rgbdpose")
    pose = cls in ("pose", "rgbdpose")
    dl = upstream_gradient(W, H, 3) * (3.0 * W * H)
    rng = np.random.default_rng(9)
    dld = rng.normal(size=(H, W)).astype(np.float32) * 0.1 if rgbd else None
    dla = rng.normal(size=(H, W)).astype(np.float32) if rgbd else None
    base = (P["pws"], P["shs"], P["alphas"], P["scales"], P["rots"], P["us"])
    if pose:
        cp = [T(sc[n]).requires_grad_() for n in ("Rcw", "tcw", "twc")]
        fn = GSFunctionFusedRGBDPose if rgbd else GSFunctionFusedPose
        out = fn.apply(*base, *cp, cam, ft)
    elif cls == "features":
        feats = T(np.random.default_rng(2).normal(size=(N, 5)).astype(np.float32)).requires_grad_()
        out = GSFunctionFusedFeatures.apply(*base, feats, cam, ft)
    else:
        out = (GSFunctionFusedRGBD if rgbd else GSFunctionFused).apply(*base, cam, ft)
    loss = (out[0] * T(dl)).sum()
    if rgbd:
        loss = loss + (out[1] * T(dld)).sum() + (out[2] * T(dla)).sum()
    loss.backward()
    torch.cuda.synchronize()
    sf, af = ops.filter3d_apply(T(sc["scales"]), T(sc["alphas"]), ft) if filt else (T(sc["scales"]), T(sc["alphas"]))
    pre = ops.preprocess(*((T(sc["pws"]), T(sc["rots"]), sf, T(sc["shs"])) + _args(sc)[4:]), alphas=af,
                         antialiased=aa, **_kw(k))
    drawn = dict(us=pre[0].cpu().numpy(), ci=pre[1].cpu().numpy(), col=pre[2].cpu().numpy(),
                 depths=pre[3].cpu().numpy(), areas=pre[4].cpu().numpy(),
                 alphas=(pre[6] if aa else af).cpu().numpy())
    camd = dict(Rcw=sc["Rcw"], tcw=sc["tcw"], twc=sc["twc"], fx=sc["fx"], fy=sc["fy"], cx=sc["cx"], cy=sc["cy"],
                width=W, height=H)
    scene = {n: sc[n] for n in ("pws", "rots", "scales", "shs", "alphas")}
    ref = ocv.step(scene, camd, rgbd=rgbd, pose=pose, aa=aa, filt=f3, dl=dl, dld=dld, dla=dla, drawn_inputs=drawn,
                   model="opencv", k=k)
    ok = ~ref["ambiguous"]
    img = out[0].detach().cpu().numpy()
    assert np.abs(img - ref["image"]).max(0)[ok].max() < 1e-4
    rows = ~ref["flagged"]
    for n in ("pws", "scales", "rots", "alphas") + (("shs",) if cls != "features" else ()):
        _close(P[n].grad.cpu().numpy(), ref["grads"][n], rows, tol=2e-4, what="d" + n)
    if pose:
        g = torch.cat([c.grad.reshape(-1) for c in cp]).cpu().numpy()
        err = np.abs(g - ref["cam_grad"]) / np.maximum(ref["absum"], 1e-30)
        assert err.max() < 2e-4


def test_graphed_and_multiview_match_the_eager_class():
    from easygaussiansplatting_b200.graphed import GraphedFusedStep
    from easygaussiansplatting_b200.parallel import MultiViewStep
    W, H, N = 160, 96, 3000
    sc = _scene(COLMAP, N, W, H, 16, seed=8)
    cam = _cam(sc, COLMAP)
    P = _params(sc)
    img, _ = GSFunctionFused.apply(P["pws"], P["shs"], P["alphas"], P["scales"], P["rots"], P["us"], cam)
    dl = T(upstream_gradient(W, H, 4))
    (img * dl).sum().backward()
    g = GraphedFusedStep(T(sc["pws"]), T(sc["shs"]), T(sc["alphas"][:, None]), T(sc["scales"]), T(sc["rots"]), cam)
    g.forward()
    assert torch.equal(g.image, img.detach())
    g.dloss_dimage.copy_(dl)
    g.backward()
    torch.cuda.synchronize()
    for n, key in (("pws", "dpws"), ("shs", "dshs"), ("scales", "dscales"), ("rots", "drots"), ("us", "dus")):
        ref = P[n].grad
        err = float((g.grads[key].reshape(ref.shape) - ref).abs().max() / ref.abs().max().clamp_min(1e-30))
        assert err <= 2e-6, (n, err)
    mv = MultiViewStep(T(sc["pws"]), T(sc["rots"]), T(sc["scales"]), T(sc["shs"]), T(sc["alphas"][:, None]))
    image, ctx = mv.render(cam)
    assert torch.equal(image, img.detach())
    mv.backward(ctx, dl, last=True)
    r = mv.reduce()
    torch.cuda.synchronize()
    for n, key in (("pws", "dpws"), ("scales", "dscales"), ("rots", "drots"), ("shs", "dshs")):
        ref = P[n].grad
        err = float((r[key].reshape(ref.shape) - ref).abs().max() / ref.abs().max().clamp_min(1e-30))
        assert err <= 2e-6, (n, err)


def test_refusals():
    from easygaussiansplatting_b200.gsfunction import GSFunction
    sc = _scene(COLMAP, 200, 64, 48, 1, seed=1)
    cam = _cam(sc, COLMAP)
    P = _params(sc)
    with pytest.raises(ValueError, match="pinhole"):
        GSFunction.apply(P["pws"], P["shs"], P["alphas"], P["scales"], P["rots"], P["us"], cam)
    with pytest.raises(ValueError, match="pinhole"):
        ops.filter3d(T(sc["pws"]), [cam])
    cam.grad_exchange = object()
    with pytest.raises(ValueError, match="pinhole"):
        GSFunctionFused.apply(P["pws"], P["shs"], P["alphas"], P["scales"], P["rots"], P["us"], cam)


def test_config2_frame():
    """1M Gaussians at 1920x1080 through COLMAP_LIKE_OPENCV: forward values and the per-Gaussian gradients
    from random moment rows, with depth, pose and AA, against the oracle"""
    sc = camera_model_scene(1 << 20, 1920, 1080, "opencv", COLMAP_LIKE_OPENCV[0], sh_dim=48, seed=0,
                            tangential_coeffs=COLMAP_LIKE_OPENCV[1])
    _per_gaussian(sc, COLMAP, True, True, True, seed=1)


def test_training_run():
    """fit a perturbed scene to a target rendered through an OPENCV camera from a hidden one: the L2 loss
    falls fourfold"""
    W, H, N = 128, 96, 1500
    sc = camera_model_scene(N, W, H, "opencv", COLMAP_LIKE_OPENCV[0], sh_dim=3, seed=11,
                            tangential_coeffs=COLMAP_LIKE_OPENCV[1])
    cam = _cam(sc, COLMAP)
    hidden = {n: T(sc[n]) for n in ("pws", "shs", "scales", "rots")}
    hidden["alphas"] = T(sc["alphas"][:, None])
    us0 = torch.zeros((N, 2), device=DEV)
    with torch.no_grad():
        target, _ = GSFunctionFused.apply(hidden["pws"], hidden["shs"], hidden["alphas"], hidden["scales"],
                                          hidden["rots"], us0, cam)
    g = torch.Generator(device=DEV).manual_seed(0)
    P = {n: v.clone() for n, v in hidden.items()}
    P["pws"] += 0.03 * torch.randn(P["pws"].shape, device=DEV, generator=g) * P["pws"].norm(dim=1, keepdim=True) / 5
    P["shs"] += 0.5 * torch.randn(P["shs"].shape, device=DEV, generator=g)
    for v in P.values():
        v.requires_grad_()
    opt = torch.optim.Adam([P["pws"], P["shs"]], lr=2e-3)
    losses = []
    for _ in range(150):
        opt.zero_grad()
        us = torch.zeros((N, 2), device=DEV, requires_grad=True)
        img, _ = GSFunctionFused.apply(P["pws"], P["shs"], P["alphas"], P["scales"], P["rots"], us, cam)
        loss = ((img - target) ** 2).mean()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert np.isfinite(losses).all()
    assert losses[-1] < losses[0] / 4, (losses[0], losses[-1])
