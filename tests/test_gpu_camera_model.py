"""The camera models (ortho, fisheye) on the H100: ops.preprocess / preprocessB against the fp64 oracle
(oracle/camera_model_oracle.py) at every SH degree with and without antialiasing, depth and the camera
gradient; pinhole through the new entry points bit-identical to the old; whole steps of the fused
classes against camera_model_oracle.step; the graphed and multi-view steps against the eager class;
the refusals; a config-2-sized frame per model; and a short fisheye training run."""
import ctypes as C

import numpy as np
import pytest
import torch

from easygaussiansplatting_b200 import _lib, ops
from easygaussiansplatting_b200.gsfunction import (Camera, GSFunctionFused, GSFunctionFusedFeatures,
                                                   GSFunctionFusedPose, GSFunctionFusedRGBD,
                                                   GSFunctionFusedRGBDPose)
from easygaussiansplatting_b200.scene import COLMAP_LIKE_FISHEYE_K, camera_model_scene, upstream_gradient
from oracle import camera_model_oracle as ocm
from oracle import oracle as orc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MODELS = [("ortho", None), ("fisheye", None), ("fisheye", COLMAP_LIKE_FISHEYE_K)]
K_FOLD = (-0.3, 0.0, 0.0, 0.0)


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _scene(model, k, N, W, H, k3, seed):
    sc = camera_model_scene(N, W, H, model, k, sh_dim=3 * k3, seed=seed)
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


def _stages(sc, model, k):
    return ocm.stages(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                      sc["fy"], sc["cx"], sc["cy"], sc["width"], sc["height"], model=model, k=k)


def _close(got, ref, rows, tol=1e-4, what=""):
    got = np.asarray(got, np.float64).reshape(len(rows), -1)[rows]
    ref = np.asarray(ref, np.float64).reshape(len(rows), -1)[rows]
    if ref.size == 0:
        return
    err = np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30)
    assert err < tol, "%s: %.3g of max|ref|" % (what, err)


def _per_gaussian(sc, model, k, k3, aa, depth, pose, seed=0, pose_only=False):
    """preprocess + preprocessB with random moment rows, against the oracle chain"""
    N = len(sc["pws"])
    args = _args(sc)
    al = T(sc["alphas"])
    pre = ops.preprocess(*args, alphas=al, antialiased=aa, camera_model=model, radial_coeffs=k)
    us, ci, col, dep, ar = (x.cpu().numpy() for x in pre[:5])
    st = _stages(sc, model, k)
    keep = st["keep"]
    thin = ocm.oaa.thin(sc["scales"])
    pc = sc["pws"].astype(np.float64) @ sc["Rcw"].astype(np.float64).T + sc["tcw"]
    band = np.abs(pc[:, 2] - 0.2) < 1e-5
    if model == "fisheye":
        band |= np.abs(ocm.fisheye_terms(pc, k)["P1"]) < 1e-4
    sure = ~band
    assert np.array_equal((dep >= 0.2)[sure], keep[sure])
    ok = keep & sure & ~thin
    _close(us, st["us"], ok, what="us")
    _close(ci, st["ci"], ok, what="conic")
    _close(col, st["col"], np.ones(N, bool), what="colour")
    s = ocm.oaa.scale(st["c2"], keep)
    if aa:
        ok &= ~ocm.oaa.flagged(sc["scales"], s)
        np.testing.assert_allclose(pre[6].cpu().numpy()[ok], (s["rho"] * sc["alphas"])[ok], rtol=1e-3)
    rng = np.random.default_rng(seed)
    m = rng.normal(size=(N, 9)).astype(np.float32)
    m[rng.random(N) < 0.1] = 0.0  # untouched Gaussians
    gz = rng.normal(size=N).astype(np.float32) if depth else None
    out = ops.preprocessB(*args, None, None, None, moments=T(m), cinv2ds=pre[1], dloss_ddepths=T(gz) if depth else None,
                          camera_grad=pose, pose_only=pose_only, antialiased=aa, alphas=al if aa else None,
                          camera_model=model, radial_coeffs=k)
    torch.cuda.synchronize()
    cig = ci.astype(np.float64)
    none = (m[:, 0] == 0) & (m[:, 1] == 0)
    gu = np.where(none[:, None], 0.0, -np.stack([cig[:, 0] * m[:, 0] + cig[:, 1] * m[:, 1],
                                                 cig[:, 1] * m[:, 0] + cig[:, 2] * m[:, 1]], 1))
    gci = np.stack([-0.5 * m[:, 2], -m[:, 3], -0.5 * m[:, 4]], 1).astype(np.float64)
    gcol, ga = m[:, 6:9].astype(np.float64), m[:, 5].astype(np.float64)
    Rcw = sc["Rcw"]
    ch = orc.chain_backward(Rcw, gu.reshape(N, 1, 2), gci.reshape(N, 1, 3), ga.reshape(N, 1, 1),
                            gcol.reshape(N, 1, 3), *st["J"])
    ref = {n: ch[n] for n in ("pws", "scales", "rots", "shs")}
    if depth:
        ref["pws"] = ref["pws"] + ocm.ordb.chain_depth(Rcw, gz.reshape(N, 1, 1), st["depths"])
    dal = ga
    per = ocm.camera_grad(st, sc["pws"], Rcw, sc["fx"], sc["fy"], sc["width"], sc["height"], gu, gci, gcol, gz,
                          model=model)["per"]
    if aa:
        gc2 = ocm.oaa.dcov2d_addend(st["c2"], keep, sc["alphas"], ga)
        add = ocm.oaa.chain(st, Rcw, gc2)
        for n in ("pws", "scales", "rots"):
            ref[n] = ref[n] + add[n]
        dal = s["rho"] * ga
        per = per + ocm.camera_grad(ocm.oaa._identity_conic(st), sc["pws"], Rcw, sc["fx"], sc["fy"], sc["width"],
                                    sc["height"], np.zeros((N, 2)), gc2, np.zeros((N, 3)), model=model)["per"]
    rows = sure & ~thin
    if aa:
        rows &= ~ocm.oaa.flagged(sc["scales"], s)
    if not pose_only:
        gpw, gsh, gs, gq, dus, dalk = (x.cpu().numpy() for x in out[:6])
        for n, got in (("pws", gpw), ("scales", gs), ("rots", gq), ("shs", gsh)):
            _close(got, ref[n], rows, what="d" + n)
        _close(dus, gu, rows, tol=1e-5, what="dus")
        _close(dalk, dal, rows, tol=1e-5, what="dalphas")
    if pose:
        g = torch.cat([x.reshape(-1) for x in out[-1]]).cpu().numpy()
        refc = per[rows].sum(0)
        err = np.abs(g - per.sum(0)) / np.maximum(np.abs(per).sum(0), 1e-30)
        assert err.max() < 1e-4, err.max()
        assert np.abs(refc).max() > 0
    return out


@pytest.mark.parametrize("model,k", MODELS)
@pytest.mark.parametrize("k3", [1, 4, 9, 16])
@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("depth,pose", [(False, False), (True, False), (False, True), (True, True)])
def test_preprocess_against_oracle(model, k, k3, aa, depth, pose):
    sc = _scene(model, k, 1000 + 37, 320, 240, k3, seed=k3)
    _per_gaussian(sc, model, k, k3, aa, depth, pose, seed=k3 + 7 * aa)


@pytest.mark.parametrize("model,k", MODELS)
@pytest.mark.parametrize("aa", [False, True])
def test_pose_only_against_oracle(model, k, aa):
    sc = _scene(model, k, 777, 320, 240, 4, seed=3)
    out = _per_gaussian(sc, model, k, 4, aa, True, True, pose_only=True)
    assert out[0] is None


@pytest.mark.parametrize("model,k", MODELS)
def test_empty_and_unaligned(model, k):
    sc = _scene(model, k, 0, 64, 48, 4, seed=1)
    pre = ops.preprocess(*_args(sc), alphas=T(sc["alphas"]), camera_model=model, radial_coeffs=k)
    assert pre[0].shape == (0, 2)
    out = ops.preprocessB(*_args(sc), None, None, None, moments=torch.zeros((0, 9), device=DEV), cinv2ds=pre[1],
                          camera_grad=True, camera_model=model, radial_coeffs=k)
    assert out[0].shape == (0, 3) and float(torch.cat([x.reshape(-1) for x in out[-1]]).abs().sum()) == 0.0
    # rows at odd float offsets (no 16-byte vector access) give the aligned results
    sc = _scene(model, k, 129, 64, 48, 4, seed=2)
    base = ops.preprocess(*_args(sc), alphas=T(sc["alphas"]), camera_model=model, radial_coeffs=k)
    rots = torch.empty((129 * 4 + 1,), device=DEV)[1:].view(129, 4)
    rots.copy_(T(sc["rots"]))
    a = list(_args(sc)); a[1] = rots
    odd = ops.preprocess(*a, alphas=T(sc["alphas"]), camera_model=model, radial_coeffs=k)
    for x, y in zip(base, odd):
        assert torch.equal(x, y)


def test_fisheye_validity_cull():
    sc = _scene("fisheye", K_FOLD, 3000, 320, 240, 1, seed=4)
    pre = ops.preprocess(*_args(sc), alphas=T(sc["alphas"]), camera_model="fisheye", radial_coeffs=K_FOLD)
    dep, ar = pre[3].cpu().numpy(), pre[4].cpu().numpy()
    pc = sc["pws"].astype(np.float64) @ sc["Rcw"].astype(np.float64).T + sc["tcw"]
    P1 = ocm.fisheye_terms(pc, K_FOLD)["P1"]
    folded = (pc[:, 2] >= 0.2) & (P1 < -1e-4)
    assert folded.sum() > 100
    assert (dep[folded] == -1).all() and (ar[folded] == 0).all()
    _per_gaussian(sc, "fisheye", K_FOLD, 1, True, True, True)
    m = torch.ones((3000, 9), device=DEV)
    g = ops.preprocessB(*_args(sc), None, None, None, moments=m, cinv2ds=pre[1], camera_model="fisheye",
                        radial_coeffs=K_FOLD)
    assert float(g[2][torch.from_numpy(folded).to(DEV)].abs().max()) == 0.0  # zero geometry gradient


def _lib_model(model, k=(0, 0, 0, 0)):
    return C.pointer(ops._CameraModel(model, (C.c_float * 4)(*k)))


@pytest.mark.parametrize("k3", [1, 4, 9, 16])
def test_pinhole_through_the_model_entry_points_is_bit_identical(k3):
    sc = _scene("pinhole", None, 1000, 320, 240, k3, seed=k3)
    sc["pws"][::17, 0] *= 6.0  # fov clamp
    sc["pws"][::23, 2] = -1.0  # culled
    args = _args(sc)
    lib = ops._L()
    N = len(sc["pws"])
    al = T(sc["alphas"])
    st = torch.cuda.current_stream().cuda_stream
    for aa in (False, True):
        ref = ops.preprocess(*args, alphas=al, antialiased=aa)
        outs = [torch.empty_like(x) for x in ref]
        p = [x.data_ptr() for x in args[:7]]
        f = [float(x) for x in args[7:]]
        rc = lib.gsb_preprocess_forward_model(N, k3, *p, *f, *[x.data_ptr() for x in outs[:5]], al.data_ptr(),
                                              outs[5].data_ptr(), outs[6].data_ptr() if aa else None,
                                              _lib_model(0), st)
        assert rc == 0
        torch.cuda.synchronize()
        for x, y in zip(ref, outs):
            assert torch.equal(x, y)
        m = T(np.random.default_rng(k3).normal(size=(N, 9)).astype(np.float32))
        gz = T(np.random.default_rng(k3 + 1).normal(size=N).astype(np.float32))
        for depth in (None, gz):
            for pose in (False, True):
                r = ops.preprocessB(*args, None, None, None, moments=m, cinv2ds=ref[1], dloss_ddepths=depth,
                                    camera_grad=pose, antialiased=aa, alphas=al if aa else None)
                o = [torch.empty_like(x) for x in r[:6]]
                gcam = torch.empty((15,), device=DEV)
                wsb = int(lib.gsb_preprocess_backward_pose_workspace_bytes(N))
                ws = torch.empty((max(wsb, 16),), dtype=torch.uint8, device=DEV)
                rc = lib.gsb_preprocess_backward_model(
                    N, k3, *p, *f, None, None, None, o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr(),
                    o[3].data_ptr(), m.data_ptr(), ref[1].data_ptr(), o[4].data_ptr(), o[5].data_ptr(),
                    depth.data_ptr() if depth is not None else None, al.data_ptr() if aa else None,
                    gcam.data_ptr() if pose else None, ws.data_ptr() if pose else None, wsb if pose else 0,
                    _lib_model(0), st)
                assert rc == 0
                torch.cuda.synchronize()
                for x, y in zip(r[:6], o):
                    assert torch.equal(x, y)
                if pose:
                    assert torch.equal(torch.cat([x.reshape(-1) for x in r[6]]), gcam)


def _cam(sc, model, k, aa=False):
    return Camera(sc["width"], sc["height"], sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(sc["Rcw"]), T(sc["tcw"]),
                  T(sc["twc"]), antialiased=aa, camera_model=model, radial_coeffs=k)


def _params(sc):
    P = {n: T(sc[n]).requires_grad_() for n in ("pws", "shs", "scales", "rots")}
    P["alphas"] = T(sc["alphas"][:, None]).requires_grad_()
    P["us"] = torch.zeros((len(sc["pws"]), 2), device=DEV, requires_grad=True)
    return P


@pytest.mark.parametrize("model,k", MODELS)
@pytest.mark.parametrize("cls", ["fused", "rgbd", "pose", "rgbdpose", "features"])
@pytest.mark.parametrize("aa,filt", [(False, False), (True, False), (False, True), (True, True)])
def test_whole_step_against_oracle(model, k, cls, aa, filt):
    W, H, N = 96, 64, 600
    sc = _scene(model, k, N, W, H, 4, seed=5)
    cam = _cam(sc, model, k, aa)
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
    # the oracle renders on the kernel's own fp32 per-Gaussian values (as the step-matrix tests do)
    sf, af = ops.filter3d_apply(T(sc["scales"]), T(sc["alphas"]), ft) if filt else (T(sc["scales"]), T(sc["alphas"]))
    pre = ops.preprocess(*((T(sc["pws"]), T(sc["rots"]), sf, T(sc["shs"])) + _args(sc)[4:]), alphas=af,
                         antialiased=aa, camera_model=model, radial_coeffs=k)
    drawn = dict(us=pre[0].cpu().numpy(), ci=pre[1].cpu().numpy(), col=pre[2].cpu().numpy(),
                 depths=pre[3].cpu().numpy(), areas=pre[4].cpu().numpy(),
                 alphas=(pre[6] if aa else af).cpu().numpy())
    camd = dict(Rcw=sc["Rcw"], tcw=sc["tcw"], twc=sc["twc"], fx=sc["fx"], fy=sc["fy"], cx=sc["cx"], cy=sc["cy"],
                width=W, height=H)
    scene = {n: sc[n] for n in ("pws", "rots", "scales", "shs", "alphas")}
    ref = ocm.step(scene, camd, rgbd=rgbd, pose=pose, aa=aa, filt=f3, dl=dl, dld=dld, dla=dla, drawn_inputs=drawn,
                   model=model, k=k)
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


@pytest.mark.parametrize("model,k", MODELS)
def test_graphed_and_multiview_match_the_eager_class(model, k):
    from easygaussiansplatting_b200.graphed import GraphedFusedStep
    from easygaussiansplatting_b200.parallel import MultiViewStep
    W, H, N = 160, 96, 3000
    sc = _scene(model, k, N, W, H, 16, seed=8)
    cam = _cam(sc, model, k)
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
    # (the gradients agree to the rasterizer backward's run-to-run rounding: its atomics add in any order)
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
    sc = _scene("fisheye", None, 200, 64, 48, 1, seed=1)
    cam = _cam(sc, "fisheye", None)
    P = _params(sc)
    with pytest.raises(ValueError, match="pinhole"):
        GSFunction.apply(P["pws"], P["shs"], P["alphas"], P["scales"], P["rots"], P["us"], cam)
    with pytest.raises(ValueError, match="pinhole"):
        ops.filter3d(T(sc["pws"]), [cam])
    cam.grad_exchange = object()
    with pytest.raises(ValueError, match="pinhole"):
        GSFunctionFused.apply(P["pws"], P["shs"], P["alphas"], P["scales"], P["rots"], P["us"], cam)


@pytest.mark.parametrize("model,k", [("ortho", None), ("fisheye", None), ("fisheye", COLMAP_LIKE_FISHEYE_K)])
def test_config2_frame(model, k):
    """1M Gaussians at 1920x1080 (the fisheye 180 degrees across): forward values and the per-Gaussian
    gradients from random moment rows, with depth, pose and AA, against the oracle"""
    sc = camera_model_scene(1 << 20, 1920, 1080, model, k, sh_dim=48, seed=0)
    _per_gaussian(sc, model, k, 16, True, True, True, seed=1)


def test_fisheye_training_run():
    """fit a perturbed scene to a fisheye target rendered from a hidden one: the L2 loss falls 4x"""
    W, H, N = 128, 96, 1500
    k = COLMAP_LIKE_FISHEYE_K
    sc = camera_model_scene(N, W, H, "fisheye", k, sh_dim=3, seed=11)
    cam = _cam(sc, "fisheye", k)
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
