"""The batch's camera gradients on the H100 (DESIGN 3.22): ops.preprocessB_batch(camera_grad=True) and
GSFunctionFusedBatch[RGBD]Pose.

- row c against ops.preprocessB(..., camera_grad=True) fed camera c's slice of the batch's own moment rows
  and conics, and against the fp64 oracle (oracle/opencv_oracle.py, which covers every camera model, with
  aa_oracle's term under antialiasing), at every camera model, SH degree, with and without antialiasing
  and depth, for C in {1, 3, 8, 64}, N not a multiple of 128 and one camera facing away from the scene;
- with pose + map the per-Gaussian outputs are gsb_preprocess_backward_batch's bits, and pose only gives
  the same camera gradients;
- pose only writes nothing per Gaussian, is run-to-run identical, and N = 0 gives C rows of zeros;
- through autograd against a lone GSFunctionFused[RGBD]Pose call per camera, with a chained twc;
- four frames of a frozen map tracked together by one pose-only optimisation."""
import math

import numpy as np
import pytest
import torch

from easygaussiansplatting_b200 import _lib, ops
from easygaussiansplatting_b200.gsfunction import (Camera, GSFunctionFusedBatchPose, GSFunctionFusedBatchRGBDPose,
                                                   GSFunctionFusedPose, GSFunctionFusedRGBDPose, camera_model_kwargs)
from easygaussiansplatting_b200.scene import synthetic_scene
from oracle import camera_model_oracle as ocm
from oracle import opencv_oracle as ocv

from test_gpu_batch import H, W, _cams, _loss_weights, _params

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
AWAY = [[-1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, -1.0]]


def n(x):
    return x.detach().cpu().numpy()


def bits(x):
    return x.detach().contiguous().view(torch.int32)


def _with_away(sc, C, model, aa):
    """_cams, with camera 1 (C >= 3) turned away from every Gaussian"""
    cams = _cams(sc, C, model, aa)
    if C >= 3:
        c = cams[1]
        R = torch.tensor(AWAY, device=DEV)
        cams[1] = Camera(W, H, c.fx, c.fy, c.cx, c.cy, R, torch.zeros(3, device=DEV), torch.zeros(3, device=DEV),
                         antialiased=aa, **camera_model_kwargs(c))
    return cams


def _moment_grads(m, ci):
    """dL/du, dL/dconic, dL/dcolour from moment rows, as the kernels convert them (fp64)"""
    m, ci = m.astype(np.float64), ci.astype(np.float64)
    none = (m[:, 0] == 0) & (m[:, 1] == 0)
    gu = -np.stack([ci[:, 0] * m[:, 0] + ci[:, 1] * m[:, 1], ci[:, 1] * m[:, 0] + ci[:, 2] * m[:, 1]], 1)
    gu[none] = 0
    gci = np.stack([-0.5 * m[:, 2], -m[:, 3], -0.5 * m[:, 4]], 1)
    return gu, gci, m[:, 6:9]


def _oracle(sc, p, cam, m, ci, gz, aa):
    """camera cam's per-Gaussian camera contributions [N,15] in fp64 from its moment rows m [N,9], the
    conics ci [N,3] they were taken on and dL/dz gz [N] (or None), and the rows the fp32 result may
    differ from them by more than rounding (near-plane band, thin, the fisheye's fold, AA's clamp)"""
    model, k = ops.camera_model_args(**camera_model_kwargs(cam))
    R, tc, tw = (n(x).astype(np.float32) for x in (cam.Rcw, cam.tcw, cam.twc))
    pws, scales, alphas = sc["pws"], n(p["scales"]), n(p["alphas"]).reshape(-1)
    st = ocv.stages(pws, n(p["rots"]), scales, n(p["shs"]), R, tc, tw, cam.fx, cam.fy, cam.cx, cam.cy, W, H,
                    model=model, k=np.asarray(k, np.float64))
    gu, gci, gcol = _moment_grads(m, ci)
    per = ocv.camera_grad(st, pws, R, cam.fx, cam.fy, W, H, gu, gci, gcol, gz, model=model)["per"]
    Nn = len(pws)
    pc = pws.astype(np.float64) @ R.astype(np.float64).T + tc
    odd = (np.abs(pc[:, 2] - 0.2) < 1e-4) | ocm.oaa.thin(scales)
    if model == "fisheye":
        odd |= np.abs(ocm.fisheye_terms(pc, k)["P1"]) < 1e-4
    if model == "opencv":
        odd |= ocv.opencv_band(pc, k, cam.fx, cam.fy, cam.cx, cam.cy, W, H)
    if aa:
        gc2 = ocm.oaa.dcov2d_addend(st["c2"], st["keep"], alphas, m[:, 5].astype(np.float64))
        per = per + ocv.camera_grad(ocm.oaa._identity_conic(st), pws, R, cam.fx, cam.fy, W, H, np.zeros((Nn, 2)), gc2,
                                    np.zeros((Nn, 3)), model=model)["per"]
        odd |= ocm.oaa.flagged(scales, ocm.oaa.scale(st["c2"], st["keep"]))
    return per, odd


def _single(p, cam, m, ci, gz, aa, pose_only=True):
    return ops.preprocessB(p["pws"], p["rots"], p["scales"], p["shs"], cam.Rcw, cam.tcw, cam.twc, cam.fx, cam.fy,
                           cam.cx, cam.cy, W, H, None, None, None, moments=m, cinv2ds=ci, dloss_ddepths=gz,
                           camera_grad=True, pose_only=pose_only, antialiased=aa, alphas=p["alphas"] if aa else None,
                           **camera_model_kwargs(cam))


def _flat(g):
    """(dRcws[C,3,3], dtcws[C,3], dtwcs[C,3]) -> [C, 15]"""
    return torch.cat([x.reshape(x.shape[0], -1) for x in g], 1)


@pytest.mark.parametrize("depth", [False, True])
@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("model", ["pinhole", "ortho", "fisheye", "opencv"])
@pytest.mark.parametrize("C", [1, 3, 8, 64])
def test_batch_camera_grad_vs_single_camera_and_oracle(C, model, aa, depth):
    for k3 in (1, 4, 9, 16):
        sc, p = _params(1037, k3, seed=3 * C + k3)
        p["alphas"] = p["alphas"].reshape(-1)
        N = p["pws"].shape[0]
        cams = _with_away(sc, C, model, aa)
        pre = ops.preprocess_batch(p["pws"], p["rots"], p["scales"], p["shs"], cams, p["alphas"])
        ci = pre[1]
        rng = np.random.default_rng(100 * C + k3)
        m = rng.normal(size=(C * N, 9)).astype(np.float32)
        m[rng.random(C * N) < 0.1] = 0.0  # untouched rows
        gz = rng.normal(size=C * N).astype(np.float32) if depth else None
        mt, gzt = torch.from_numpy(m).to(DEV), torch.from_numpy(gz).to(DEV) if depth else None
        kw = dict(dloss_ddepths=gzt, alphas=p["alphas"] if aa else None)
        both = ops.preprocessB_batch(p["pws"], p["rots"], p["scales"], p["shs"], cams, mt, ci, camera_grad=True, **kw)
        G = n(_flat(both[6])).astype(np.float64)
        assert G.shape == (C, 15)
        # pose + map: the map outputs are the plain batch backward's bits; pose only: the same camera rows
        base = ops.preprocessB_batch(p["pws"], p["rots"], p["scales"], p["shs"], cams, mt, ci, **kw)
        for a, b in zip(both[:6], base):
            assert torch.equal(bits(a), bits(b))
        po = ops.preprocessB_batch(p["pws"], p["rots"], p["scales"], p["shs"], cams, mt, ci, camera_grad=True,
                                   pose_only=True, **kw)
        assert all(x is None for x in po[:6])
        assert torch.equal(bits(_flat(po[6])), bits(_flat(both[6])))
        for c, cam in enumerate(cams):
            mc, gzc = mt[c * N:(c + 1) * N], gzt[c * N:(c + 1) * N] if depth else None
            one = n(torch.cat([x.reshape(-1) for x in _single(p, cam, mc, ci[c], gzc, aa)[-1]])).astype(np.float64)
            per, odd = _oracle(sc, p, cam, m[c * N:(c + 1) * N], n(ci[c]), gz[c * N:(c + 1) * N] if depth else None, aa)
            absum = np.abs(per).sum(0)
            # the single-camera call: its bits up to the compiler's contraction of the lens (fisheye, DESIGN 3.21)
            rel = 1e-5 if model == "fisheye" else 1e-6
            assert (np.abs(G[c] - one) <= rel * absum).all(), (k3, c, np.abs(G[c] - one) / np.maximum(absum, 1e-30))
            # the fp64 oracle: test_gpu_pose's 1e-5 (the models: their single-camera tests' 1e-4), and 1e-3 of the
            # rows fp32 may put on the other side of a cull, clamp or AA clamp
            rel = 1e-5 if model == "pinhole" else 1e-4
            tol = rel * absum + 1e-3 * np.abs(per[odd]).sum(0)
            err = np.abs(G[c] - per.sum(0))
            assert (err <= tol).all(), (k3, c, err / np.maximum(absum, 1e-30))
            if C >= 3 and c == 1:  # facing away: nothing projects, only the colour branch (SH degree > 0)
                assert not G[c, :12].any()


def test_pose_only_writes_nothing_is_reproducible_and_n0_gives_zeros():
    lib = _lib.load()
    C, k3 = 8, 16
    sc, p = _params(20001, k3, seed=7)
    N = p["pws"].shape[0]
    cams = _with_away(sc, C, "pinhole", False)
    bc = ops.BatchCameras(cams, torch.device(DEV))
    pre = ops.preprocess_batch(p["pws"], p["rots"], p["scales"], p["shs"], bc, p["alphas"])
    g = torch.Generator(device=DEV).manual_seed(0)
    mom = torch.randn((C * N, 9), generator=g, device=DEV)
    gz = torch.randn((C * N,), generator=g, device=DEV)
    inputs = [p["pws"], p["rots"], p["scales"], p["shs"], bc.poses, mom, pre[1], gz]
    keep = [x.clone() for x in inputs]
    wsb = lib.gsb_preprocess_backward_batch_pose_workspace_bytes(C, N)
    assert wsb == C * ((N + 127) // 128) * 64
    ws = torch.full((wsb // 4 + 64,), float("nan"), device=DEV)
    out = torch.full((C * 15 + 32,), 7.0, device=DEV)
    P = lambda t: t.data_ptr()
    runs = []
    for _ in range(2):
        _lib.check(lib.gsb_preprocess_backward_batch_pose(
            C, N, k3, P(p["pws"]), P(p["rots"]), P(p["scales"]), P(p["shs"]), *bc.args(), P(mom), P(pre[1]), P(gz),
            None, *([None] * 6), P(out), P(ws), wsb, None), lib)
        torch.cuda.synchronize()
        runs.append(out.clone())
    assert torch.equal(bits(runs[0]), bits(runs[1]))
    assert (out[C * 15:] == 7.0).all() and torch.isnan(ws[wsb // 4:]).all()
    for a, b in zip(inputs, keep):
        assert torch.equal(bits(a), bits(b))
    # pose + map: every per-Gaussian output (pre-filled with a sentinel) is written, the camera rows are the same
    full = [torch.full(s, float("nan"), device=DEV) for s in ((N, 3), (N, 3 * k3), (N, 3), (N, 4), (C, N, 2), (N,))]
    g2 = torch.full((C * 15,), float("nan"), device=DEV)
    _lib.check(lib.gsb_preprocess_backward_batch_pose(
        C, N, k3, P(p["pws"]), P(p["rots"]), P(p["scales"]), P(p["shs"]), *bc.args(), P(mom), P(pre[1]), P(gz),
        None, *[P(x) for x in full], P(g2), P(ws), wsb, None), lib)
    torch.cuda.synchronize()
    assert torch.equal(bits(g2), bits(runs[0][:C * 15]))
    assert all(not torch.isnan(x).any() for x in full)
    # N = 0: C rows of zeros, no workspace
    z = torch.full((C * 15,), float("nan"), device=DEV)
    assert lib.gsb_preprocess_backward_batch_pose_workspace_bytes(C, 0) == 0
    _lib.check(lib.gsb_preprocess_backward_batch_pose(
        C, 0, k3, *([None] * 4), bc.poses.data_ptr(), bc.intrinsics.data_ptr(), bc.model_id, float(W), float(H),
        *([None] * 10), P(z), None, 0, None), lib)
    torch.cuda.synchronize()
    assert torch.equal(bits(z), torch.zeros(C * 15, dtype=torch.int32, device=DEV))


def _leaves(p, need_map):
    L = {k: p[k].clone().requires_grad_(need_map) for k in ("pws", "shs", "scales", "rots")}
    L["alphas"] = p["alphas"].reshape(-1, 1).clone().requires_grad_(need_map)
    return L


@pytest.mark.parametrize("need_map", [True, False])
@pytest.mark.parametrize("rgbd", [False, True])
@pytest.mark.parametrize("model,aa", [("pinhole", False), ("pinhole", True), ("opencv", False), ("fisheye", True)])
def test_autograd_pose_classes_against_a_lone_call_per_camera(model, aa, rgbd, need_map):
    C = 3
    sc, p = _params(2000, 16, seed=31)
    cams = _with_away(sc, C, model, aa)
    N = p["pws"].shape[0]
    Gi, Gd, Ga = _loss_weights(C, 5)
    chain = not need_map  # twc = -R^T t built in torch: autograd chains it into Rcws and tcws
    L = _leaves(p, need_map)
    Rs = torch.stack([c.Rcw for c in cams]).requires_grad_()
    ts = torch.stack([c.tcw for c in cams]).requires_grad_()
    ws = -(Rs.transpose(1, 2) @ ts[:, :, None])[:, :, 0] if chain else \
        torch.stack([c.twc for c in cams]).clone().requires_grad_()
    us = torch.zeros((C, N, 2), device=DEV, requires_grad=need_map)
    args = (L["pws"], L["shs"], L["alphas"], L["scales"], L["rots"], us, Rs, ts, ws, cams)
    if rgbd:
        img, dep, alp, mask = GSFunctionFusedBatchRGBDPose.apply(*args)
        ((img * Gi).sum() + (dep * Gd).sum() + (alp * Ga).sum()).backward()
    else:
        img, mask = GSFunctionFusedBatchPose.apply(*args)
        (img * Gi).sum().backward()
    assert mask.shape == (C, N)
    S = _leaves(p, need_map)
    for c, cam in enumerate(cams):
        R = cam.Rcw.clone().requires_grad_()
        t = cam.tcw.clone().requires_grad_()
        w = -(R.t() @ t) if chain else cam.twc.clone().requires_grad_()
        u = torch.zeros((N, 2), device=DEV, requires_grad=need_map)
        a = (S["pws"], S["shs"], S["alphas"], S["scales"], S["rots"], u, R, t, w, cam)
        if rgbd:
            i1, d1, a1, _ = GSFunctionFusedRGBDPose.apply(*a)
            ((i1 * Gi[c]).sum() + (d1 * Gd[c]).sum() + (a1 * Ga[c]).sum()).backward()
            planes = ((img, i1), (dep, d1), (alp, a1))
        else:
            i1, _ = GSFunctionFusedPose.apply(*a)
            (i1 * Gi[c]).sum().backward()
            planes = ((img, i1),)
        for x, y in planes:
            if model == "fisheye":
                assert torch.allclose(x[c].detach(), y.detach(), rtol=0, atol=5e-3)
            else:
                assert torch.equal(x[c].detach(), y.detach())
        # the pose: within 1e-5 of sum_i |c_i| (fisheye: 1e-3, as its map gradients), the contributions taken
        # from the oracle on the lone call's own moment rows (the two rasterizer backwards add them in
        # different orders)
        a = _absum(sc, p, cam, rgbd, aa, Gi[c], Gd[c], Ga[c])
        rel = 1e-3 if model == "fisheye" else 1e-5
        wR, wt = n(R.grad).astype(np.float64), n(t.grad).astype(np.float64)
        if chain:
            tR, Rm = np.abs(n(t)).astype(np.float64), np.abs(n(R)).astype(np.float64)
            tolR = rel * (a[:9].reshape(3, 3) + np.outer(tR, a[12:])) + 1e-6 * np.abs(wR)
            tolt = rel * (a[9:12] + Rm @ a[12:]) + 1e-6 * np.abs(wt)
        else:
            tolR, tolt = rel * a[:9].reshape(3, 3), rel * a[9:12]
            assert (np.abs(n(ws.grad[c]) - n(w.grad)) <= rel * a[12:]).all(), c
        assert (np.abs(n(Rs.grad[c]) - wR) <= tolR).all(), c
        assert (np.abs(n(ts.grad[c]) - wt) <= tolt).all(), c
    if need_map:
        rel = 1e-3 if model == "fisheye" else 1e-5
        for k in ("pws", "shs", "alphas", "scales", "rots"):
            tol = rel * max(float(S[k].grad.abs().max()), 1e-30)
            assert float((L[k].grad - S[k].grad).abs().max()) <= tol, k
    else:
        assert all(L[k].grad is None for k in L) and us.grad is None


def _pre1(p, cam):
    return ops.preprocess(p["pws"], p["rots"], p["scales"], p["shs"], cam.Rcw, cam.tcw, cam.twc, cam.fx, cam.fy,
                          cam.cx, cam.cy, W, H, alphas=p["alphas"].reshape(-1), antialiased=cam.antialiased,
                          **camera_model_kwargs(cam))


def _absum(sc, p, cam, rgbd, aa, dl, dld, dla):
    """sum_i |c_i| of cam's camera gradient under the upstream planes, from the oracle on the moment rows of
    cam's single frame drawn as GSFunctionFused[RGBD] draws it"""
    pre = _pre1(p, cam)
    drawn = pre[6] if aa else p["alphas"].reshape(-1)
    d = pre[3].clone()
    if rgbd:
        fr = ops.splat_rgbd(H, W, pre[0], pre[1], drawn, d, pre[2], pre[4].clone(), records=pre[5])
        mom, dz = ops.splatB_rgbd(H, W, pre[0], pre[1], drawn, d, pre[2], fr[1], fr[2], fr[3], fr[4], dl, dld, dla,
                                  moments_only=True)[:2]
        dz = n(dz)
    else:
        fr = ops.splat(H, W, pre[0], pre[1], drawn, d, pre[2], pre[4].clone(), records=pre[5])
        mom = ops.splatB(H, W, pre[0], pre[1], drawn, d, pre[2], fr[1], fr[2], fr[3], fr[4], dl, moments_only=True)
        dz = None
    per, _ = _oracle(sc, p, cam, n(mom), n(pre[1]), dz, aa)
    return np.abs(per).sum(0)


# ---------------------------------------------------------------- tracking several frames
def _hat(xi):
    w, v = xi[:3], xi[3:]
    z = torch.zeros((), device=xi.device)
    return torch.stack([torch.stack([z, -w[2], w[1], v[0]]), torch.stack([w[2], z, -w[0], v[1]]),
                        torch.stack([-w[1], w[0], z, v[2]]), torch.stack([z, z, z, z])])


def test_rgbd_tracking_of_four_frames_in_one_pose_only_batch():
    """a frozen map; four frames, each started 1 degree (about its own oblique axis) and 2 cm off, found
    together by Adam on L1(image) + L1(depth) through one GSFunctionFusedBatchRGBDPose call per step, each
    pose an se(3) tangent through torch.matrix_exp (test_gpu_pose's tracking, batched)"""
    Nn, Wt, Ht, C = 20000, 640, 360, 4
    sc = synthetic_scene(Nn, Wt, Ht, sh_dim=48, seed=4)
    sc["scales"] = (sc["scales"] * 3.0).astype(np.float32)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    G = [T(sc[k]) for k in ("pws", "shs")] + [T(sc["alphas"][:, None])] + [T(sc[k]) for k in ("scales", "rots")]
    G.append(torch.zeros((C, Nn, 2), device=DEV))
    Rt, tt, cams = [], [], []
    for c in range(C):
        a = 0.05 - 0.03 * c
        R = torch.tensor([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]], device=DEV)
        t = torch.tensor([0.05 - 0.02 * c, -0.03 + 0.01 * c, 0.1], device=DEV)
        Rt.append(R)
        tt.append(t)
        cams.append(Camera(Wt, Ht, sc["fx"], sc["fy"], sc["cx"], sc["cy"], R, t, -(R.t() @ t)))
    Rt, tt = torch.stack(Rt), torch.stack(tt)

    def render(R, t):
        return GSFunctionFusedBatchRGBDPose.apply(*G, R, t, -(R.transpose(1, 2) @ t[:, :, None])[:, :, 0], cams)

    with torch.no_grad():
        img_gt, dep_gt = [x.clone() for x in render(Rt, tt)[:2]]
    axes = torch.tensor([[0.3, -0.8, 0.5], [-0.6, 0.2, 0.7], [0.5, 0.5, -0.7], [0.1, 0.9, 0.4]], device=DEV)
    axes = axes / axes.norm(dim=1, keepdim=True)
    shifts = torch.tensor([[0.02, 0, 0], [0, 0.02, 0], [0, 0, 0.02], [-0.02, 0, 0]], device=DEV)
    T0 = []
    c_gt = -(Rt.transpose(1, 2) @ tt[:, :, None])[:, :, 0]
    for c in range(C):
        dR = torch.linalg.matrix_exp(_hat(torch.cat([axes[c] * math.radians(1.0), torch.zeros(3, device=DEV)]))[:3, :3])
        R0 = dR @ Rt[c]
        M = torch.eye(4, device=DEV)
        M[:3, :3] = R0
        M[:3, 3] = -(R0 @ (c_gt[c] + shifts[c]))
        T0.append(M)

    def errors(c, M):
        R, t = M[:3, :3], M[:3, 3]
        cosang = ((torch.trace(R @ Rt[c].t()) - 1) / 2).clamp(-1, 1)
        return torch.acos(cosang).item(), (-(R.t() @ t) - c_gt[c]).norm().item()

    e0 = [errors(c, T0[c]) for c in range(C)]
    for er, et in e0:
        assert abs(er - math.radians(1.0)) < 1e-4 and abs(et - 0.02) < 1e-5
    xi = torch.zeros((C, 6), device=DEV, requires_grad=True)
    opt = torch.optim.Adam([xi], lr=2e-3)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=0.985)
    for _ in range(200):
        Ms = torch.stack([torch.linalg.matrix_exp(_hat(xi[c])) @ T0[c] for c in range(C)])
        img, dep = render(Ms[:, :3, :3], Ms[:, :3, 3])[:2]
        loss = (img - img_gt).abs().mean() + (dep - dep_gt).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        sched.step()
    with torch.no_grad():
        for c in range(C):
            er, et = errors(c, torch.linalg.matrix_exp(_hat(xi[c])) @ T0[c])
            print("frame %d: rotation %.3g -> %.3g rad, centre %.3g -> %.3g" % (c, e0[c][0], er, e0[c][1], et))
            assert er < 0.1 * e0[c][0] and et < 0.1 * e0[c][1], (c, er, et)
