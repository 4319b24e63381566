"""Batched rendering on the H100 (DESIGN 3.21): ops.preprocess_batch / splat_batch / splatB_batch /
preprocessB_batch and GSFunctionFusedBatch[RGBD] against C single-camera calls.

- the per-Gaussian outputs of camera c, its tile patch lists (record ids c N + n -> n) and its planes are
  the single-camera call's bits, at every camera model, SH degree, with and without antialiasing, at a
  frame whose width and height are not multiples of 16;
- the map gradients equal the sum of the C single-camera gradients within 1e-5 of each tensor's
  max |g|, and dL/du[c] camera c's;
- a camera facing away from every Gaussian, between cameras whose Gaussians straddle their frames'
  edges, renders zeros and gets no gradient;
- the capacity path, and a call that outgrows it;
- a short training run at C = 4 against the loop of single-camera steps."""
import math

import numpy as np
import pytest
import torch

from easygaussiansplatting_b200 import ops
from easygaussiansplatting_b200.gsfunction import (Camera, GSFunctionFused, GSFunctionFusedBatch,
                                                   GSFunctionFusedBatchRGBD, GSFunctionFusedRGBD, camera_model_kwargs)
from easygaussiansplatting_b200.scene import ring_camera, synthetic_scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
W, H = 83, 61  # not multiples of 16: partial tiles and 3 pad rows per frame
LENS = {"pinhole": None, "ortho": None, "fisheye": (0.05, -0.01, 0.002, -0.0005), "opencv": (-0.12, 0.03)}


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _params(N, k3, seed):
    sc = synthetic_scene(N, W, H, sh_dim=3 * k3, seed=seed)
    return sc, {k: T(sc[k]) for k in ("pws", "shs", "scales", "rots", "alphas")}


def _cams(sc, C, model="pinhole", aa=False):
    """C distinct poses and intrinsics (and lens coefficients) of one size and model"""
    cams = []
    for c in range(C):
        R, t, tw = ring_camera(c, C, radius=0.3)
        f = 1.0 + 0.04 * c
        kw = {}
        if model == "ortho":
            fx, fy = 25.0 * f, 24.0 * f
        else:
            fx, fy = sc["fx"] * f, sc["fy"] * (1.0 + 0.03 * c)
        if model == "fisheye":
            kw["radial_coeffs"] = tuple(x * (1.0 + 0.1 * c) for x in LENS["fisheye"])
        elif model == "opencv":
            kw["radial_coeffs"] = tuple(x * (1.0 + 0.1 * c) for x in LENS["opencv"])
            kw["tangential_coeffs"] = (2e-4 * c, -3e-4)
        cams.append(Camera(W, H, fx, fy, sc["cx"] + 0.7 * c, sc["cy"] - 0.4 * c, T(R), T(t), T(tw), antialiased=aa,
                           camera_model=model, **kw))
    return cams


def _single_pre(p, cam):
    return ops.preprocess(p["pws"], p["rots"], p["scales"], p["shs"], cam.Rcw, cam.tcw, cam.twc, cam.fx, cam.fy,
                          cam.cx, cam.cy, cam.width, cam.height, alphas=p["alphas"], antialiased=cam.antialiased,
                          **camera_model_kwargs(cam))


def _same(a, b, model, what):
    """the bits of the single-camera call.  FISHEYE: within rtol 1e-5 / atol 1e-4 (see DESIGN 3.21: ptxas
    contracts one more multiply-add of its lens into an FFMA in the camera loop; the last-bit change of
    fx s x shows as many ulp of a mean u near 0)"""
    if model == "fisheye" and a.dtype == torch.float32:
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-4, equal_nan=True), (what, float((a - b).abs().nan_to_num().max()))
    else:
        assert torch.equal(a, b), what


def _tile_lists(ranges, gsid, t0, T_, shift):
    return [gsid[int(ranges[t, 0]):int(ranges[t, 1])] - shift if ranges[t, 1] > ranges[t, 0] else gsid[:0]
            for t in range(t0, t0 + T_)]


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("model", ["pinhole", "ortho", "fisheye", "opencv"])
@pytest.mark.parametrize("C", [1, 3, 8])
def test_batch_forward_is_the_single_camera_calls_bit_for_bit(C, model, aa):
    for k3 in (1, 4, 9, 16):
        sc, p = _params(1500, k3, seed=10 * C + k3)
        cams = _cams(sc, C, model, aa)
        pre = ops.preprocess_batch(p["pws"], p["rots"], p["scales"], p["shs"], cams, p["alphas"])
        N = p["pws"].shape[0]
        singles = [_single_pre(p, cam) for cam in cams]
        for c, s in enumerate(singles):
            for i in range(5):  # us, cinv2ds, colors, depths, areas
                _same(pre[i][c], s[i], model, (k3, c, i))
            rb = pre[5][c * N:(c + 1) * N].clone()
            ids = rb[:, 2].view(torch.int32)
            assert torch.equal(ids, torch.arange(c * N, (c + 1) * N, device=DEV, dtype=torch.int32))
            rs = s[5].clone()
            rb[:, 2] = 0.0
            rs[:, 2] = 0.0
            _same(rb, rs, model, (k3, c))
            if aa:
                _same(pre[6][c], s[6], model, (k3, c))
        drawn_b = pre[6] if aa else p["alphas"].expand(C, N).contiguous()
        # camera c's single frame from the batch's own per-Gaussian rows (ids c N + n -> n)
        own = []
        for c in range(C):
            rc = pre[5][c * N:(c + 1) * N].clone()
            rc[:, 2] = torch.arange(N, device=DEV, dtype=torch.int32).view(torch.float32)
            own.append((pre[0][c].clone(), pre[1][c].clone(), drawn_b[c].clone(), pre[3][c].clone(), pre[2][c].clone(),
                        pre[4][c].clone(), rc))
        out = ops.splat_batch(H, W, pre[0], pre[1], drawn_b, pre[3], pre[2], pre[4], records=pre[5], rgbd=True)
        Tn = ops._tiles(H, W)
        assert out[3].shape == (C * Tn, 2) and out[0].shape == (C, 3, H, W) and out[5].shape == (C, H, W)
        assert int(out[4].numel()) > 0
        for c, o in enumerate(own):
            ref = ops.splat_rgbd(H, W, *o[:6], records=o[6])
            for i in (0, 1, 2, 5, 6):  # image, contrib, final_tau, depth, alpha
                assert torch.equal(out[i][c], ref[i]), (k3, c, i)
            lb = _tile_lists(out[3].cpu(), out[4], c * Tn, Tn, c * N)
            ls = _tile_lists(ref[3].cpu(), ref[4], 0, Tn, 0)
            assert all(torch.equal(a, b) for a, b in zip(lb, ls)), (k3, c)
            # the in-place culls of the binning: the same depths / areas
            assert torch.equal(pre[3][c], o[3]) and torch.equal(pre[4][c], o[5])


def _loss_weights(C, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn((C, 3, H, W), generator=g, device=DEV), torch.randn((C, H, W), generator=g, device=DEV),
            torch.randn((C, H, W), generator=g, device=DEV))


def _leaves(p):
    return {k: p[k].clone().requires_grad_() for k in ("pws", "shs", "scales", "rots")} | \
        {"alphas": p["alphas"][:, None].clone().requires_grad_()}


def _close(a, b, what, rel=1e-5):
    tol = rel * max(float(b.abs().max()), 1e-30)
    err = float((a - b).abs().max())
    assert err <= tol, "%s: max err %g > %g" % (what, err, tol)


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("rgbd", [False, True])
@pytest.mark.parametrize("aa,model", [(False, "pinhole"), (True, "pinhole"), (False, "opencv"), (True, "fisheye")])
@pytest.mark.parametrize("C", [1, 3, 8])
def test_batch_backward_is_the_sum_of_the_single_camera_gradients(C, aa, model, rgbd, filtered):
    sc, p = _params(2000, 16, seed=C + 7)
    cams = _cams(sc, C, model, aa)
    N = p["pws"].shape[0]
    f3d = ops.filter3d(p["pws"], _cams(sc, 2)) if filtered else None
    Gi, Gd, Ga = _loss_weights(C, 3)
    # batched
    L = _leaves(p)
    us = torch.zeros((C, N, 2), device=DEV, requires_grad=True)
    args = (L["pws"], L["shs"], L["alphas"], L["scales"], L["rots"], us, cams, f3d)
    if rgbd:
        img, dep, alp, mask = GSFunctionFusedBatchRGBD.apply(*args)
        loss = (img * Gi).sum() + (dep * Gd).sum() + (alp * Ga).sum()
    else:
        img, mask = GSFunctionFusedBatch.apply(*args)
        loss = (img * Gi).sum()
    loss.backward()
    assert mask.shape == (C, N)
    # the loop of single-camera calls
    S = _leaves(p)
    dus = []
    for c, cam in enumerate(cams):
        u = torch.zeros((N, 2), device=DEV, requires_grad=True)
        a = (S["pws"], S["shs"], S["alphas"], S["scales"], S["rots"], u, cam, f3d)
        if rgbd:
            i1, d1, a1, m1 = GSFunctionFusedRGBD.apply(*a)
            lc = (i1 * Gi[c]).sum() + (d1 * Gd[c]).sum() + (a1 * Ga[c]).sum()
        else:
            i1, m1 = GSFunctionFused.apply(*a)
            lc = (i1 * Gi[c]).sum()
        lc.backward()
        assert torch.equal(mask[c], m1)
        planes = ((img, i1), (dep, d1), (alp, a1)) if rgbd else ((img, i1),)
        for x, y in planes:
            if model == "fisheye":  # (see _same; a last-bit change of a mean can flip a pixel's alpha' skip)
                assert torch.allclose(x[c], y.detach(), rtol=0, atol=5e-3)
            else:
                assert torch.equal(x[c], y.detach())
        dus.append(u.grad)
    rel = 1e-3 if model == "fisheye" else 1e-5  # (fisheye: see above)
    for k in ("pws", "shs", "alphas", "scales", "rots"):
        _close(L[k].grad, S[k].grad, k, rel)
    for c in range(C):
        _close(us.grad[c], dus[c], "dus[%d]" % c, rel)


def test_batch_isolation_camera_facing_away_and_edge_gaussians():
    """cameras 0 and 2 see Gaussians straddling their top and bottom edges and pad rows (some huge);
    camera 1, between them, faces away from all of them"""
    sc, p = _params(3000, 16, seed=5)
    rng = np.random.default_rng(1)
    N = p["pws"].shape[0]
    # pull a third of the Gaussians onto the top / bottom frame edges, and make some of them huge
    pws = sc["pws"].copy()
    idx = rng.choice(N, N // 3, replace=False)
    z = pws[idx, 2]
    v = np.where(rng.random(idx.size) < 0.5, rng.uniform(-3, 3, idx.size), H + rng.uniform(-3, 3, idx.size))
    pws[idx, 1] = (v - sc["cy"]) * z / sc["fy"]
    scales = sc["scales"].copy()
    scales[idx[:40]] *= 30.0
    p["pws"], p["scales"] = T(pws), T(scales)
    base = _cams(sc, 1)[0]
    away = torch.tensor([[-1.0, 0, 0], [0, 1, 0], [0, 0, -1]], device=DEV)
    cams = [base, Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], away, torch.zeros(3, device=DEV)),
            Camera(W, H, sc["fx"] * 1.1, sc["fy"] * 1.1, sc["cx"] + 2, sc["cy"] - 1, base.Rcw, base.tcw)]
    L = _leaves(p)
    us = torch.zeros((3, N, 2), device=DEV, requires_grad=True)
    img, dep, alp, mask = GSFunctionFusedBatchRGBD.apply(L["pws"], L["shs"], L["alphas"], L["scales"], L["rots"], us,
                                                         cams)
    (img.square().sum() + dep.sum() + alp.sum()).backward()
    assert not mask[1].any()
    img, dep, alp = img.detach(), dep.detach(), alp.detach()
    assert float(img[1].abs().max()) == 0.0 and float(dep[1].abs().max()) == 0.0 and float(alp[1].abs().max()) == 0.0
    assert float(us.grad[1].abs().max()) == 0.0
    for c in (0, 2):
        assert float(alp[c, 0].max()) > 0 and float(alp[c, H - 1].max()) > 0  # the edge rows are covered
        s = _single_pre(p, cams[c])
        ref = ops.splat_rgbd(H, W, s[0], s[1], p["alphas"], s[3], s[2], s[4], records=s[5])
        for i, t in ((0, img), (5, dep), (6, alp)):
            assert torch.equal(t[c].detach(), ref[i]), (c, i)


def test_batch_capacity_path_and_outgrown_capacity():
    sc, p = _params(4000, 4, seed=2)
    cams = _cams(sc, 4)
    N = p["pws"].shape[0]
    pre = ops.preprocess_batch(p["pws"], p["rots"], p["scales"], p["shs"], cams, p["alphas"])

    def frame(capacity):
        d, a = pre[3].clone(), pre[4].clone()
        return ops.splat_batch(H, W, pre[0], pre[1], p["alphas"], d, pre[2], a, records=pre[5], capacity=capacity)

    exact = frame(False)
    key = ("batch", torch.device(DEV).index, 4, H, W, N)
    ops._CAPACITY.pop(key, None)
    frame(True)  # learns the bounds
    stats = dict(ops.CAPACITY_STATS)
    cap = frame(True)
    assert ops.CAPACITY_STATS["capacity_frames"] == stats["capacity_frames"] + 1
    for a, b in zip(exact, cap):
        assert torch.equal(a, b)
    ops._CAPACITY[key] = (16, ops._CAPACITY[key][1])  # far too few patch slots: redone the exact way
    out = frame(True)
    assert ops.CAPACITY_STATS["outgrown"] == stats["outgrown"] + 1
    for a, b in zip(exact, out):
        assert torch.equal(a, b)


def test_batch_training_lowers_the_loss_like_the_loop():
    C, steps = 4, 40
    sc, target = _params(3000, 16, seed=11)
    cams = _cams(sc, C)
    with torch.no_grad():
        N = target["pws"].shape[0]
        gt, _ = GSFunctionFusedBatch.apply(target["pws"], target["shs"], target["alphas"][:, None], target["scales"],
                                           target["rots"], torch.zeros((C, N, 2), device=DEV), cams)
    g = torch.Generator(device=DEV).manual_seed(0)
    start = {k: v + 0.05 * torch.randn(v.shape, generator=g, device=DEV) * v.abs().mean() for k, v in target.items()}
    start["alphas"] = target["alphas"].clamp(0.05, 0.9)

    def run(batched):
        L = _leaves(start)
        opt = torch.optim.Adam(list(L.values()), lr=2e-3)
        losses = []
        for _ in range(steps):
            opt.zero_grad()
            if batched:
                img, _ = GSFunctionFusedBatch.apply(L["pws"], L["shs"], L["alphas"], L["scales"], L["rots"],
                                                    torch.zeros((C, N, 2), device=DEV, requires_grad=True), cams)
                loss = (img - gt).abs().mean()
            else:
                loss = 0.0
                for c, cam in enumerate(cams):
                    img, _ = GSFunctionFused.apply(L["pws"], L["shs"], L["alphas"], L["scales"], L["rots"],
                                                   torch.zeros((N, 2), device=DEV, requires_grad=True), cam)
                    loss = loss + (img - gt[c]).abs().mean() / C
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
        return losses

    lb, ll = run(True), run(False)
    assert math.isclose(lb[0], ll[0], rel_tol=1e-5)
    assert lb[-1] < 0.9 * lb[0] and ll[-1] < 0.9 * ll[0]
    assert abs(lb[-1] - ll[-1]) <= 0.05 * ll[-1]
