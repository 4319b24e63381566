"""The intrinsics gradient on the GPU (DESIGN 3.23): gsb_preprocess_backward_intrinsics and its batch form
against the fp64 oracle, the pose entry point, the map-only backward and each other; the autograd classes'
`intrinsics` argument; and recovering a perturbed OPENCV calibration with a frozen map."""
import numpy as np
import pytest
import torch

from oracle import aa_oracle as oaa
from oracle import intrinsics_oracle as oin
from oracle import opencv_oracle as ocv
from easygaussiansplatting_b200 import ops
from easygaussiansplatting_b200.gsfunction import (Camera, GSFunctionFusedBatchPose, GSFunctionFusedBatchRGBDPose,
                                                   GSFunctionFusedPose, GSFunctionFusedRGBDPose)

pytestmark = pytest.mark.gpu
DEV = "cuda"
W, H = 320, 240
KS = {"pinhole": (0.0, 0.0, 0.0, 0.0), "ortho": (0.0, 0.0, 0.0, 0.0), "fisheye": (0.05, -0.01, 0.004, -0.001),
      "opencv": (-0.08, 0.02, 0.001, -0.002)}


def _scene(N, k3, seed, model, away=False):
    rng = np.random.default_rng(seed)
    z = rng.uniform(1.5, 6.0, N)
    span = 0.15 if model == "ortho" else 0.6
    a, b = rng.uniform(-span, span, N), rng.uniform(-span, span, N) * 0.75
    if model != "ortho":
        n = N // 8  # past the 1.3 tan_fov clamp bound (about 0.8 of x/z), and near the axis (fisheye's series)
        a[:n] = np.sign(rng.normal(size=n)) * rng.uniform(0.9, 1.1, n)
        a[n:2 * n] = rng.uniform(-0.015, 0.015, n)
        b[n:2 * n] = rng.uniform(-0.015, 0.015, n)
    pw = np.stack([a * (1 if model == "ortho" else z), b * (1 if model == "ortho" else z), z], 1)
    if away:
        pw[:, 2] = -pw[:, 2]
    q = rng.normal(size=(N, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    s = rng.uniform(0.01, 0.08, (N, 3)) * (0.2 if model == "ortho" else 1)
    sh = rng.normal(size=(N, 3 * k3)) * 0.3
    a = rng.uniform(0.3, 0.9, N)
    f = 90.0 if model == "ortho" else 260.0
    intr = [f, f * 0.98, W / 2 + 3, H / 2 - 2] + list(KS[model])
    th = 0.05
    R = np.array([[np.cos(th), 0, np.sin(th)], [0, 1, 0], [-np.sin(th), 0, np.cos(th)]])
    t = np.array([0.05, -0.02, 0.1])
    f32 = lambda x: torch.tensor(np.asarray(x), dtype=torch.float32, device=DEV)
    return dict(pws=f32(pw), rots=f32(q), scales=f32(s), shs=f32(sh), alphas=f32(a), R=f32(R), t=f32(t),
                twc=f32(-R.T @ t), intr=intr, model=model)


def _kw(sc):
    k = sc["intr"][4:]
    m = sc["model"]
    return dict(camera_model=m, radial_coeffs=(k[:2] if m == "opencv" else k) if m in ("opencv", "fisheye") else None,
                tangential_coeffs=k[2:] if m == "opencv" else None)


def _fwd(sc, aa):
    i = sc["intr"]
    return ops.preprocess(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["R"], sc["t"], sc["twc"], i[0], i[1], i[2],
                          i[3], W, H, alphas=sc["alphas"], antialiased=aa, **_kw(sc))


def _bwd(sc, aa, moments, cinv, dz, **kw):
    i = sc["intr"]
    return ops.preprocessB(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["R"], sc["t"], sc["twc"], i[0], i[1],
                           i[2], i[3], W, H, None, None, None, moments=moments, cinv2ds=cinv, dloss_ddepths=dz,
                           antialiased=aa, alphas=sc["alphas"] if aa else None, **_kw(sc), **kw)


def _moments(N, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    m = torch.randn((N, 9), generator=g) * torch.tensor([3, 3, 30, 30, 30, 1, 1, 1, 1.0])
    return m.to(DEV), (torch.randn((N,), generator=g) * 0.5).to(DEV)


def _oracle(sc, aa, moments, cinv, depths):
    f64 = lambda x: x.detach().double().cpu().numpy()
    pw, q, s = f64(sc["pws"]), f64(sc["rots"]), f64(sc["scales"])
    R = f64(sc["R"])
    pc = np.empty_like(pw)  # as camera_point rounds it: each fmaf an exact product and one fp32 rounding
    for r in range(3):
        acc = f64(sc["t"])[r] + 0 * pw[:, 0]
        for c in (2, 1, 0):
            acc = (R[r, c] * pw[:, c] + acc).astype(np.float32).astype(np.float64)
        pc[:, r] = acc
    keep = f64(depths) != -1.0
    pc = np.where(keep[:, None], pc, [0.0, 0.0, 1.0])
    w, x, y, z = q.T
    Rq = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                   2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                   2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
    M = Rq * s[:, None, :]
    S = M @ M.transpose(0, 2, 1)
    c3 = S[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]
    intr = [float(np.float32(v)) for v in sc["intr"]]
    lim = oin.limits(sc["model"], intr, W, H)
    gu, gcon, ga = oin.kernel_upstream(f64(moments), f64(cinv))
    add = None
    if aa:
        c2 = oin._cov2d(oin.dproj(pc, sc["model"], intr, lim)[1], R, c3)[0]
        add = oaa.dcov2d_addend(c2, keep, f64(sc["alphas"]), ga)
    return oin.per_gaussian(pc, R, c3, sc["model"], intr, lim, gu, gcon, add, keep)


@pytest.mark.parametrize("k3", [1, 4, 9, 16])
@pytest.mark.parametrize("depth", [False, True])
@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("model", oin.MODELS)
def test_single_camera_against_oracle(model, aa, depth, k3):
    N = 1037
    sc = _scene(N, k3, 11 + k3, model)
    pre = _fwd(sc, aa)
    cinv, depths = pre[1], pre[3]
    mom, dz = _moments(N, k3 + 3)
    out = _bwd(sc, aa, mom, cinv, dz if depth else None, camera_grad=True, pose_only=True, intrinsics_grad=True)
    got = out[-1].double().cpu().numpy()
    per = _oracle(sc, aa, mom, cinv, depths)
    tol = (1e-5 if model == "pinhole" else 1e-4) * np.abs(per).sum(0) + 1e-30
    assert (np.abs(got - per.sum(0)) <= tol).all(), (got, per.sum(0), tol)
    if model in ("pinhole", "ortho"):
        assert not got[4:].any()
    # two runs give the same bits
    again = _bwd(sc, aa, mom, cinv, dz if depth else None, camera_grad=True, pose_only=True, intrinsics_grad=True)
    assert torch.equal(again[-1], out[-1]) and torch.equal(again[-2][0], out[-2][0])


@pytest.mark.parametrize("model", oin.MODELS)
def test_facing_away_and_empty(model):
    sc = _scene(300, 16, 5, model, away=True)
    pre = _fwd(sc, False)
    mom, _ = _moments(300, 1)
    out = _bwd(sc, False, mom, pre[1], None, camera_grad=True, pose_only=True, intrinsics_grad=True)
    assert not out[-1].any()
    e = _scene(0, 16, 5, model)
    z9, z3 = torch.zeros((0, 9), device=DEV), torch.zeros((0, 3), device=DEV)
    out = _bwd(e, False, z9, z3, None, camera_grad=True, pose_only=True, intrinsics_grad=True)
    assert not out[-1].any() and out[-1].shape == (8,)


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("model", oin.MODELS)
def test_pose_columns_and_map_gradients(model, aa):
    N = 2000
    sc = _scene(N, 16, 3, model)
    pre = _fwd(sc, aa)
    mom, dz = _moments(N, 9)
    both = _bwd(sc, aa, mom, pre[1], dz, camera_grad=True, intrinsics_grad=True)
    pose = _bwd(sc, aa, mom, pre[1], dz, camera_grad=True)
    plain = _bwd(sc, aa, mom, pre[1], dz)
    for a, b in zip(both[:6], plain[:6]):
        assert torch.equal(a, b)
    gi = torch.cat([x.reshape(-1) for x in both[6]])
    gp = torch.cat([x.reshape(-1) for x in pose[6]])
    print("pose columns bit-identical to gsb_preprocess_backward_pose (%s, aa=%s): %s" % (model, aa, torch.equal(gi, gp)))
    # within 1e-6 sum_i |c_i|, the per-Gaussian pose contributions' magnitudes (fp64 oracle)
    absum = _pose_absum(sc, aa, mom, pre[1], dz)
    assert ((gi - gp).abs().double().cpu().numpy() <= 1e-6 * absum).all(), ((gi - gp).abs(), absum)


def _pose_absum(sc, aa, moments, cinv, dz):
    """sum over the Gaussians of |each one's 15 pose contributions| from the fp64 oracle (camera_grad of
    opencv_oracle.stages, plus antialiasing's dcov2d term as step_oracle adds it)"""
    f = lambda x: x.detach().double().cpu().numpy()
    i = sc["intr"]
    k = np.asarray(i[4:], np.float64) if sc["model"] in ("fisheye", "opencv") else None
    st = ocv.stages(f(sc["pws"]), f(sc["rots"]), f(sc["scales"]), f(sc["shs"]), f(sc["R"]), f(sc["t"]), f(sc["twc"]),
                    i[0], i[1], i[2], i[3], W, H, model=sc["model"], k=k)
    gu, gcon, ga = oin.kernel_upstream(f(moments), f(cinv))
    m = f(moments)
    per = ocv.camera_grad(st, f(sc["pws"]), f(sc["R"]), i[0], i[1], W, H, gu, gcon, m[:, 6:9], f(dz),
                          model=sc["model"])["per"]
    if aa:
        gc2 = oaa.dcov2d_addend(st["c2"], st["keep"], f(sc["alphas"]), ga)
        N = len(ga)
        per = per + ocv.camera_grad(oaa._identity_conic(st), f(sc["pws"]), f(sc["R"]), i[0], i[1], W, H,
                                    np.zeros((N, 2)), gc2, np.zeros((N, 3)), model=sc["model"])["per"]
    return np.abs(per).sum(0)


def _cams(sc, Cn, seed):
    rng = np.random.default_rng(seed)
    cams, rows = [], []
    for c in range(Cn):
        i = list(sc["intr"])
        i[0] *= 1 + 0.02 * rng.normal(); i[1] *= 1 + 0.02 * rng.normal()
        i[2] += rng.normal(); i[3] += rng.normal()
        th = 0.03 * rng.normal()
        R = torch.tensor([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]], dtype=torch.float32,
                         device=DEV) @ sc["R"]
        t = sc["t"] + torch.tensor(rng.normal(size=3) * 0.02, dtype=torch.float32, device=DEV)
        kw = _kw(dict(sc, intr=i))
        cams.append(Camera(W, H, i[0], i[1], i[2], i[3], R, t, -R.T @ t, **kw))
        rows.append(i)
    return cams, rows


@pytest.mark.parametrize("Cn,k3", [(1, 9), (3, 9), (8, 9), (64, 9), (64, 16)])
@pytest.mark.parametrize("model", oin.MODELS)
def test_batch_rows_match_single_calls(model, Cn, k3):
    """row c of the batch against the single call for camera c; C = 64 at SH degree 3 needs the kernel's
    largest shared memory (the SH tile plus 64 cameras' partial rows, above 48 KB)"""
    N = 700
    sc = _scene(N, k3, 21, model)
    cams, _ = _cams(sc, Cn, Cn)
    bc = ops.BatchCameras(cams, DEV)
    pre = ops.preprocess_batch(sc["pws"], sc["rots"], sc["scales"], sc["shs"], bc, sc["alphas"])
    mom, _ = _moments(Cn * N, Cn)
    out = ops.preprocessB_batch(sc["pws"], sc["rots"], sc["scales"], sc["shs"], bc, mom, pre[1], camera_grad=True,
                                pose_only=True, intrinsics_grad=True)
    gint = out[-1]
    for c in range(Cn):
        cam = cams[c]
        one = ops.preprocessB(sc["pws"], sc["rots"], sc["scales"], sc["shs"], cam.Rcw, cam.tcw, cam.twc, cam.fx,
                              cam.fy, cam.cx, cam.cy, W, H, None, None, None, moments=mom[c * N:(c + 1) * N],
                              cinv2ds=pre[1][c], camera_grad=True, pose_only=True, intrinsics_grad=True,
                              camera_model=cam.camera_model, radial_coeffs=cam.radial_coeffs,
                              tangential_coeffs=cam.tangential_coeffs)
        tol = (1e-5 if model == "fisheye" else 1e-6) * float(one[-1].abs().sum()) + 1e-30
        assert (gint[c] - one[-1]).abs().max() <= tol, (c, gint[c], one[-1])
        g15 = torch.cat([x.reshape(-1) for x in one[-2]])
        assert torch.allclose(torch.cat([x[c].reshape(-1) for x in out[-2]]), g15, rtol=1e-5,
                              atol=1e-6 * float(g15.abs().sum()))


@pytest.mark.parametrize("intr_dev", ["cpu", "cuda"])
@pytest.mark.parametrize("rgbd", [False, True])
def test_autograd_single_every_combination(rgbd, intr_dev):
    sc = _scene(1500, 16, 4, "opencv")
    N = 1500
    cam = Camera(W, H, *sc["intr"][:4], sc["R"], sc["t"], sc["twc"], antialiased=True, **_kw(sc))
    f3d = torch.full((N,), 1e-3, device=DEV)
    ref = None
    for need_map in (False, True):
        for need_pose in (False, True):
            for need_intr in (False, True):
                if not (need_map or need_pose or need_intr):
                    continue
                P = [sc[k].clone().requires_grad_(need_map) for k in ("pws", "shs")]
                al = sc["alphas"][:, None].clone().requires_grad_(need_map)
                S = [sc[k].clone().requires_grad_(need_map) for k in ("scales", "rots")]
                us = torch.zeros((N, 2), device=DEV, requires_grad=need_map)
                uabs = torch.zeros((N, 2), device=DEV, requires_grad=need_map)
                pose = [x.clone().requires_grad_(need_pose) for x in (sc["R"], sc["t"], sc["twc"])]
                intr = torch.tensor(sc["intr"], dtype=torch.float32, device=intr_dev, requires_grad=need_intr)
                cls = GSFunctionFusedRGBDPose if rgbd else GSFunctionFusedPose
                outs = cls.apply(P[0], P[1], al, S[0], S[1], us, *pose, cam, f3d, uabs, intr)
                loss = outs[0].square().sum() + (outs[1].sum() * 0.01 if rgbd else 0)
                loss.backward()
                if need_intr:
                    assert intr.grad.device.type == intr_dev and intr.grad.abs().sum() > 0
                    if ref is None:
                        ref = intr.grad.cpu().clone()
                    else:
                        assert torch.allclose(intr.grad.cpu(), ref, rtol=1e-5, atol=1e-6 * float(ref.abs().sum()))
                else:
                    assert intr.grad is None
                assert (P[0].grad is not None) == need_map and (pose[0].grad is not None) == need_pose


@pytest.mark.parametrize("intr_dev", ["cpu", "cuda"])
@pytest.mark.parametrize("rgbd", [False, True])
def test_autograd_batch_every_combination(rgbd, intr_dev):
    """GSFunctionFusedBatch[RGBD]Pose with intrinsics, for every needs_input_grad combination of map, poses
    and intrinsics: each requested gradient is there and no other; the intrinsics gradient of camera c equals
    the single-camera class's for that camera alone (the loss is a sum over the cameras); the map and pose
    gradients agree, to rounding, whether or not the intrinsics are differentiated"""
    N, Cn = 1200, 3
    sc = _scene(N, 9, 14, "opencv")
    cams, rows = _cams(sc, Cn, 6)
    cams = [Camera(W, H, c.fx, c.fy, c.cx, c.cy, c.Rcw, c.tcw, c.twc, antialiased=True, camera_model="opencv",
                   radial_coeffs=c.radial_coeffs, tangential_coeffs=c.tangential_coeffs) for c in cams]
    cls1 = GSFunctionFusedRGBDPose if rgbd else GSFunctionFusedPose
    clsb = GSFunctionFusedBatchRGBDPose if rgbd else GSFunctionFusedBatchPose

    def loss(outs):
        return outs[0].square().sum() + (outs[1].sum() * 0.01 if rgbd else 0)

    # per camera, the single class: the reference intrinsics gradient
    single = []
    for c, cam in enumerate(cams):
        intr = torch.tensor(rows[c], dtype=torch.float32, device=intr_dev, requires_grad=True)
        outs = cls1.apply(sc["pws"], sc["shs"], sc["alphas"][:, None], sc["scales"], sc["rots"],
                          torch.zeros((N, 2), device=DEV), cam.Rcw, cam.tcw, cam.twc, cam, None, None, intr)
        loss(outs).backward()
        single.append(intr.grad.cpu())
    single = torch.stack(single)
    seen = {}
    for need_map in (False, True):
        for need_pose in (False, True):
            for need_intr in (False, True):
                if not (need_map or need_pose or need_intr):
                    continue
                P = [sc[k].clone().requires_grad_(need_map) for k in ("pws", "shs")]
                al = sc["alphas"][:, None].clone().requires_grad_(need_map)
                S = [sc[k].clone().requires_grad_(need_map) for k in ("scales", "rots")]
                us = torch.zeros((Cn, N, 2), device=DEV, requires_grad=need_map)
                pose = [torch.stack([getattr(c, a) for c in cams]).clone().requires_grad_(need_pose)
                        for a in ("Rcw", "tcw", "twc")]
                intr = torch.tensor(rows, dtype=torch.float32, device=intr_dev, requires_grad=need_intr)
                outs = clsb.apply(P[0], P[1], al, S[0], S[1], us, *pose, cams, None, intr)
                loss(outs).backward()
                assert (intr.grad is not None) == need_intr and (P[0].grad is not None) == need_map
                assert (pose[0].grad is not None) == need_pose
                if need_intr:
                    assert intr.grad.device.type == intr_dev
                    g = intr.grad.cpu()
                    assert (((g - single).abs()) <= 1e-5 * single.abs().sum(1, keepdim=True)).all(), (g, single)
                # each combination is a new forward and rasterizer backward, whose moment sums are not
                # bit-reproducible, and the pose comes from the pose or the pose + intrinsics kernel: the
                # same gradients to rounding (the bits for fixed moment rows: test_pose_columns_and_map_gradients)
                for key, v in (("map", P[0].grad), ("pose", pose[0].grad)):
                    if v is not None:
                        if key in seen:
                            assert torch.allclose(seen[key], v, rtol=1e-4, atol=1e-5 * float(v.abs().max())), key
                        seen[key] = v.clone()


def test_autograd_batch_shared_camera():
    sc = _scene(1200, 4, 8, "fisheye")
    cams, _ = _cams(sc, 3, 2)
    N = 1200
    base = torch.tensor(sc["intr"], dtype=torch.float32, requires_grad=True)
    intr = base[None].expand(3, 8)
    Rs = torch.stack([c.Rcw for c in cams]); ts = torch.stack([c.tcw for c in cams])
    ws = torch.stack([c.twc for c in cams])
    us = torch.zeros((3, N, 2), device=DEV)
    img, _ = GSFunctionFusedBatchPose.apply(sc["pws"], sc["shs"], sc["alphas"][:, None], sc["scales"], sc["rots"], us,
                                            Rs, ts, ws, cams, None, intr)
    img.square().sum().backward()
    assert base.grad is not None and base.grad[:4].abs().min() > 0


def test_calibration_recovery_with_frozen_map():
    """render an OPENCV scene from true intrinsics, start from nominal ones, fit the intrinsics alone"""
    rng = np.random.default_rng(0)
    N, Cn = 6000, 4
    sc = _scene(N, 1, 30, "opencv")
    sc["scales"] = sc["scales"] * 0.6
    sc["shs"] = torch.tensor(rng.uniform(-1.5, 1.5, (N, 3)), dtype=torch.float32, device=DEV)
    nominal = [260.0, 260.0, W / 2, H / 2, 0.0, 0.0, 0.0, 0.0]
    true = [260.0 * 1.02, 260.0 * 1.02, W / 2 + 3, H / 2 - 2, -0.08, 0.0, 0.0, 0.0]
    cams = []
    for c in range(Cn):
        th = 0.08 * (c - 1.5)
        R = torch.tensor([[np.cos(th), 0, np.sin(th)], [0, 1, 0], [-np.sin(th), 0, np.cos(th)]], dtype=torch.float32,
                         device=DEV)
        t = torch.tensor([0.1 * (c - 1.5), 0.0, 0.2], dtype=torch.float32, device=DEV)
        cams.append(Camera(W, H, *nominal[:4], R, t, -R.T @ t, camera_model="opencv"))
    Rs = torch.stack([c.Rcw for c in cams]); ts = torch.stack([c.tcw for c in cams])
    ws = torch.stack([c.twc for c in cams])
    us = torch.zeros((Cn, N, 2), device=DEV)
    args = (sc["pws"], sc["shs"], sc["alphas"][:, None], sc["scales"], sc["rots"], us, Rs, ts, ws, cams, None)
    with torch.no_grad():
        gt, _ = GSFunctionFusedBatchPose.apply(*args, torch.tensor(true)[None].expand(Cn, 8))
    # one physical camera: fx, fy, cx, cy, k1, shared by the views
    scale = torch.tensor([100.0, 100.0, 10.0, 10.0, 0.1])
    x = (torch.tensor(nominal[:5]) / scale).requires_grad_(True)
    opt = torch.optim.Adam([x], lr=2e-3)
    err0 = np.abs(np.array(nominal[:5]) - np.array(true[:5]))
    for _ in range(300):
        opt.zero_grad()
        v = x * scale
        intr = torch.cat([v, torch.zeros(3)])[None].expand(Cn, 8)
        img, _ = GSFunctionFusedBatchPose.apply(*args, intr)
        (img - gt).abs().mean().backward()
        opt.step()
    err = np.abs((x * scale).detach().numpy() - np.array(true[:5]))
    print("calibration errors before", err0, "after", err)
    assert (err <= err0 / 10).all(), (err0, err)
