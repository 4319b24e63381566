"""Absolute-gradient densification (AbsGS) on the GPU: the _abs rasterizers (k_draw_bwd_abs,
k_draw_bwd_rgbd_abs) through `splatB(..., absgrad=True)` / `splatB_rgbd(..., absgrad=True)`, the C
entry points, the fused autograd classes' `us_abs` input and DensityController fed `us_abs.grad`.

1. Identities: every other output of the _abs calls (the four tensors, the moment rows, dL/dz) is
   that of the plain call, to the order of its float atomics.
2. Oracle parity: dloss_dus_abs against oracle/absgrad_oracle.c (fp64, on the same fp32 inputs) at
   1e-4 of max|ref| off threshold-ambiguous Gaussians and 5e-3 on them, at odd frame sizes, the
   schedule-edge scenes of test_gpu_parity.py, the opacity clamp, N = 0 and P = 0, the capacity
   path and its fallback, records given / cached / re-packed, an output at an odd 4-byte offset and
   BASELINE config 2; the RGB-D form with depth-only and alpha-only upstream gradients.
3. The four fused classes with and without antialiasing and the 3D filter; refusals.
4. Density control on the statistic, and a short training run that densifies on it."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import absgrad_oracle as oabs
from oracle import density_oracle as do
from oracle import oracle as orc
from oracle import rgbd_oracle as orgbd
from easygaussiansplatting_b200.scene import synthetic_scene, upstream_gradient

from test_gpu_parity import (DEV, boundary_frame, boundary_scene, clamp_scene, dense_scene, gaussians_in_tile, n,
                             op_inputs, scene_with_culls, stage_pipeline, t)
from test_gpu_rgbd import bound, preprocess, upstream

pytestmark = pytest.mark.gpu


def ops():
    from easygaussiansplatting_b200 import ops as o
    return o


def lib():
    from easygaussiansplatting_b200 import _lib
    return _lib.load()


def close(a, b, name, rel=1e-5):
    """equal to the order of float atomics: max |a - b| <= rel max |b|"""
    assert a.shape == b.shape, (name, a.shape, b.shape)
    if b.numel() == 0:
        return
    a, b = a.double(), b.double()
    err, s = float((a - b).abs().max()), float(b.abs().max())
    assert err <= rel * max(s, 1e-30), "%s: %.3e of %.3e" % (name, err, s)


def launches(name):
    L = lib()
    ids = [L.gsb_profile_kernel_name(i).decode() for i in range(L.gsb_profile_kernels())]
    return L.gsb_profile_launches(ids.index(name))


def check_abs(H, W, us_d, ci_d, al_d, d_d, col_d, ar_d, seed=0, records=None, capacity=False, rgbd=True,
              tol_scale=1.0):
    """the colour (and, with rgbd, the RGB-D) backward with absgrad against the plain calls and the
    oracle.  d_d / ar_d are not modified.  -> the colour call's five tensors"""
    o = ops()
    us, ci, col, al = n(us_d), n(ci_d), n(col_d), n(al_d)
    d_in, a_in = n(d_d).copy(), n(ar_d).copy()
    d1, a1 = d_d.clone(), ar_d.clone()
    out = o.splat(H, W, us_d, ci_d, al_d, d1, col_d, a1, records=records, capacity=capacity)
    ref = orc.splat(H, W, us, ci, al, d_in.copy(), col, a_in.copy(), margin=2e-5 * tol_scale)
    assert np.array_equal(n(out[4]), ref["gsid"])
    dl = upstream_gradient(W, H, seed) * (3.0 * W * H)
    g4 = o.splatB(H, W, us_d, ci_d, al_d, d1, col_d, *out[1:5], t(dl), records=records)
    n_abs = launches("draw_backward_abs")
    g5 = o.splatB(H, W, us_d, ci_d, al_d, d1, col_d, *out[1:5], t(dl), records=records, absgrad=True)
    assert len(g5) == 5 and g5[4].shape == (us.shape[0], 2) and g5[4].dtype == torch.float32
    if out[4].numel():
        assert launches("draw_backward_abs") == n_abs + 1
    for a, b, name in zip(g5[:4], g4, ("dus", "dcinv2ds", "dalphas", "dcolors")):
        close(a, b, name)
    m = o.splatB(H, W, us_d, ci_d, al_d, d1, col_d, *out[1:5], t(dl), moments_only=True, records=records)
    m2, dabs2 = o.splatB(H, W, us_d, ci_d, al_d, d1, col_d, *out[1:5], t(dl), moments_only=True, records=records,
                         absgrad=True)
    close(m2, m, "moment rows")
    close(dabs2, g5[4], "absgrad, moment form")
    du_o, dabs_o, amb = oabs.splat_backward_abs(H, W, us, ci, al, col, ref, dl, margin=2e-5 * tol_scale)
    assert amb.mean() <= 0.01 * tol_scale
    bound(g5[4], dabs_o, amb, "absgrad", 1e-4 * tol_scale, 5e-3 * tol_scale)
    bound(g5[0], du_o, amb, "dus", 1e-4 * tol_scale, 5e-3 * tol_scale)
    assert (n(g5[4]) >= 0).all()
    touched = np.zeros(us.shape[0], bool)
    touched[ref["gsid"]] = True
    assert not n(g5[4])[~touched].any()  # exact zeros where nothing replays the Gaussian
    if rgbd:
        d2, a2 = d_d.clone(), ar_d.clone()
        out5 = o.splat_rgbd(H, W, us_d, ci_d, al_d, d2, col_d, a2, records=records, capacity=capacity)
        ref5 = orgbd.splat_rgbd(H, W, us, ci, al, d_in.copy(), col, a_in.copy(), margin=2e-5 * tol_scale)
        zmax = max(float(np.abs(ref5["z"][ref5["gsid"]]).max(initial=0.0)), 1.0)
        dl3, dld, dla = upstream(W, H, seed, zmax)
        plain = o.splatB_rgbd(H, W, us_d, ci_d, al_d, d2, col_d, *out5[1:5], t(dl3), t(dld), t(dla), records=records)
        g6 = o.splatB_rgbd(H, W, us_d, ci_d, al_d, d2, col_d, *out5[1:5], t(dl3), t(dld), t(dla), records=records,
                           absgrad=True)
        assert len(g6) == 6
        for a, b, name in zip(g6[:5], plain, ("dus", "dcinv2ds", "dalphas", "dcolors", "ddepths")):
            close(a, b, "rgbd " + name)
        mm, dz, dabs3 = o.splatB_rgbd(H, W, us_d, ci_d, al_d, d2, col_d, *out5[1:5], t(dl3), t(dld), t(dla),
                                      moments_only=True, records=records, absgrad=True)
        close(dz, plain[4], "rgbd ddepths, moment form")
        close(dabs3, g6[5], "rgbd absgrad, moment form")
        _, dabs_o5, amb5 = oabs.splat_backward_rgbd_abs(H, W, us, ci, al, col, ref5["z"], ref5, dl3, dld, dla,
                                                        margin=2e-5 * tol_scale)
        bound(g6[5], dabs_o5, amb5, "rgbd absgrad", 1e-4 * tol_scale, 5e-3 * tol_scale)
    return g5


# ---------------------------------------------------------------- 2. oracle parity
@pytest.mark.parametrize("N,W,H", [(3000, 979, 546), (2000, 255, 131), (40, 17, 9), (8, 7, 5)])
def test_absgrad_vs_oracle_odd_frames(N, W, H):
    sc = scene_with_culls(N, W, H, 3, N)
    us, ci, col, d, ar = preprocess(sc)
    check_abs(H, W, us, ci, t(sc["alphas"]), d, col, ar, seed=N)


def test_absgrad_schedule_edges_empty_whole_and_dense_tiles():
    """boundary_scene: empty tiles, whole-tile (<= 32 patches) and four-entry tiles at the chunk
    edges, partial phase-B flushes and opacities above the clamp; the dense early-termination scene"""
    parts, expect, _, _ = boundary_scene(np.random.default_rng(7))
    W, H = boundary_frame(expect)
    check_abs(H, W, *op_inputs(parts), seed=7)
    sc = dense_scene()
    o = stage_pipeline(sc, calc_J=False)
    check_abs(sc["height"], sc["width"], o["us"], o["cinv2ds"], t(sc["alphas"]), o["depths"], o["colors"],
              o["areas"], seed=11)


def test_absgrad_clamped_opacity():
    sc = clamp_scene()
    o = stage_pipeline(sc, calc_J=False)
    assert (sc["alphas"] > 0.99).any()
    check_abs(sc["height"], sc["width"], o["us"], o["cinv2ds"], t(sc["alphas"]), o["depths"], o["colors"],
              o["areas"], seed=2)
    # whole tiles of clamped records at the 32-record edges
    rng = np.random.default_rng(9)
    parts = []
    for i, k in enumerate([31, 32, 33, 64, 65]):
        p = gaussians_in_tile(i, 0, k, rng, alpha=(0.5, 1.0))
        p[2][::3] = 1.0
        parts.append(p)
    check_abs(16, 16 * 5, *op_inputs(parts), seed=9)


def test_absgrad_empty_scene_and_no_patches():
    o = ops()
    W, H = 100, 70
    e = torch.empty((0, 2), device=DEV)
    z3, z1 = torch.empty((0, 3), device=DEV), torch.empty(0, device=DEV)
    out = o.splat_rgbd(H, W, e, z3, z1, z1, z3, torch.empty((0, 2), dtype=torch.int32, device=DEV))
    g = o.splatB(H, W, e, z3, z1, z1, z3, *out[1:5], torch.ones((3, H, W), device=DEV), absgrad=True)
    assert g[4].shape == (0, 2)
    g = o.splatB_rgbd(H, W, e, z3, z1, z1, z3, *out[1:5], torch.ones((3, H, W), device=DEV),
                      torch.ones((H, W), device=DEV), torch.ones((H, W), device=DEV), absgrad=True)
    assert g[5].shape == (0, 2)
    # every Gaussian behind the camera: P = 0, all zeros
    sc = synthetic_scene(500, W, H, sh_dim=3, seed=1)
    sc["pws"][:, 2] = -1.0
    us, ci, col, d, ar = preprocess(sc)
    al = t(sc["alphas"])
    out = o.splat_rgbd(H, W, us, ci, al, d, col, ar)
    assert out[4].numel() == 0
    g = o.splatB(H, W, us, ci, al, d, col, *out[1:5], torch.ones((3, H, W), device=DEV), absgrad=True)
    assert all(not bool(x.any()) for x in g)
    g = o.splatB_rgbd(H, W, us, ci, al, d, col, *out[1:5], torch.ones((3, H, W), device=DEV),
                      torch.ones((H, W), device=DEV), torch.ones((H, W), device=DEV), absgrad=True)
    assert all(not bool(x.any()) for x in g)


def test_absgrad_capacity_path_and_overflow_fallback():
    o = ops()
    N, W, H = 30000, 800, 600
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=8)
    us, ci, col, d, ar = preprocess(sc)
    al = t(sc["alphas"])
    key = (torch.device(DEV).index or 0, H, W, N)
    o._CAPACITY.pop(key, None)
    exact = check_abs(H, W, us, ci, al, d, col, ar, seed=8, capacity=True, rgbd=False)
    assert key in o._CAPACITY
    cap = check_abs(H, W, us, ci, al, d, col, ar, seed=8, capacity=True)
    close(cap[4], exact[4], "capacity frame")
    o._CAPACITY[key] = (64, o._CAPACITY[key][1])  # far too few patch slots: redone the exact way
    before = o.CAPACITY_STATS["outgrown"]
    over = check_abs(H, W, us, ci, al, d, col, ar, seed=8, capacity=True, rgbd=False)
    assert o.CAPACITY_STATS["outgrown"] == before + 1
    close(over[4], exact[4], "fallback frame")


def test_absgrad_records_given_cached_and_repacked():
    o = ops()
    N, W, H = 20000, 640, 480
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=5)
    p = {k: t(sc[k]) for k in ("pws", "rots", "scales", "shs", "Rcw", "tcw", "twc")}
    al = t(sc["alphas"])
    us, ci, col, d, ar, rec = o.preprocess(p["pws"], p["rots"], p["scales"], p["shs"], p["Rcw"], p["tcw"], p["twc"],
                                           sc["fx"], sc["fy"], sc["cx"], sc["cy"], W, H, alphas=al)
    given = check_abs(H, W, us, ci, al, d, col, ar, seed=5, records=rec)
    cached = check_abs(H, W, us, ci, al, d, col, ar, seed=5)  # splat attached its records to gsid
    close(cached[4], given[4], "cached records")
    # re-packed: the records dropped from gsid
    out = o.splat(H, W, us, ci, al, d.clone(), col, ar.clone())
    o.forget_records(out[4])
    dl = t(upstream_gradient(W, H, 5) * (3.0 * W * H))
    repacked = o.splatB(H, W, us, ci, al, d, col, *out[1:5], dl, absgrad=True)
    close(repacked[4], given[4], "re-packed records")


def test_absgrad_c_entry_point_at_odd_offsets():
    """gsb_splat_backward_abs / _rgbd_abs with dloss_dus_abs one float into its buffer (scalar
    atomics at any 4-byte boundary) and the moment rows given: the output of ops.splatB"""
    o, L = ops(), lib()
    N, W, H = 5001, 333, 211
    sc = scene_with_culls(N, W, H, 3, 41)
    us, ci, col, d, ar = preprocess(sc)
    al = t(sc["alphas"])
    out = o.splat_rgbd(H, W, us, ci, al, d, col, ar)
    P = out[4].numel()
    dl = t(upstream_gradient(W, H, 41) * (3.0 * W * H))
    dld, dla = torch.randn((H, W), device=DEV), torch.randn((H, W), device=DEV)
    want = o.splatB(H, W, us, ci, al, d, col, *out[1:5], dl, absgrad=True)[4]
    want5 = o.splatB_rgbd(H, W, us, ci, al, d, col, *out[1:5], dl, dld, dla, absgrad=True)[5]
    ws = torch.empty(L.gsb_splat_backward_workspace_bytes(N, H, W, P) + 1, dtype=torch.uint8, device=DEV)
    mom = torch.empty(N * 9 + 1, device=DEV)[1:]
    dz = torch.empty(N + 1, device=DEV)[1:]
    for rgbd in (False, True):
        buf = torch.full((2 * N + 1,), float("nan"), device=DEV)
        dabs = buf[1:]
        assert dabs.data_ptr() % 8 == 4
        common = [C.c_void_p(x.data_ptr()) for x in (us, ci, al, col)]
        fr = [C.c_void_p(x.data_ptr()) for x in (out[1], out[2], out[3], out[4], dl)]
        stream = torch.cuda.current_stream().cuda_stream
        if rgbd:
            rc = L.gsb_splat_backward_rgbd_abs(H, W, N, P, *common, d.data_ptr(), *fr, dld.data_ptr(), dla.data_ptr(),
                                               None, ws.data_ptr() + 1, ws.numel() - 1, None, None, None, None,
                                               mom.data_ptr(), dz.data_ptr(), dabs.data_ptr(), stream)
        else:
            rc = L.gsb_splat_backward_abs(H, W, N, P, *common, *fr, None, ws.data_ptr() + 1, ws.numel() - 1, None,
                                          None, None, None, mom.data_ptr(), dabs.data_ptr(), stream)
        assert rc == 0, L.gsb_last_error()
        assert bool(torch.isfinite(dabs).all()) and float(buf[0].item()) != float(buf[0].item())  # NaN kept
        close(dabs.view(N, 2), want5 if rgbd else want, "odd offset, rgbd=%s" % rgbd)


def test_absgrad_rgbd_depth_only_and_alpha_only():
    o = ops()
    N, W, H = 3000, 979, 546
    sc = scene_with_culls(N, W, H, 3, 31)
    us, ci, col, d, ar = preprocess(sc)
    al = t(sc["alphas"])
    d0, ar0 = n(d).copy(), n(ar).copy()
    out = o.splat_rgbd(H, W, us, ci, al, d, col, ar)
    ref = orgbd.splat_rgbd(H, W, n(us), n(ci), n(al), d0, n(col), ar0)
    zmax = max(float(np.abs(ref["z"][ref["gsid"]]).max()), 1.0)
    dl, dld, dla = upstream(W, H, 31, zmax)
    zero = np.zeros_like(dld)
    for a, b in ((dld, zero), (zero, dla)):
        g = o.splatB_rgbd(H, W, us, ci, al, d, col, *out[1:5], t(np.zeros_like(dl)), t(a), t(b), absgrad=True)
        _, want, amb = oabs.splat_backward_rgbd_abs(H, W, n(us), n(ci), n(al), n(col), ref["z"], ref,
                                                    np.zeros_like(dl), a, b)
        assert float(g[5].max()) > 0 and want.max() > 0
        bound(g[5], want, amb, "absgrad from one plane")


def test_absgrad_config2_vs_oracle():
    """1M Gaussians at 1920x1080 (BASELINE config 2)"""
    N, W, H = 1_000_000, 1920, 1080
    sc = synthetic_scene(N, W, H, sh_dim=48, seed=0)
    us, ci, col, d, ar = preprocess(sc)
    check_abs(H, W, us, ci, t(sc["alphas"]), d, col, ar, seed=2, rgbd=False)


# ---------------------------------------------------------------- 3. autograd classes
def _class_frame(seed=12, N=6000, W=241, H=163):
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=seed)
    P = {k: t(sc[k]) for k in ("pws", "shs", "scales", "rots")}
    P["alphas"] = t(sc["alphas"][:, None])
    return sc, P, W, H


def _ops_absgrad(sc, P, W, H, aa, f3, rgbd, pose, grads):
    """what the classes compute, through the operators: the frame as _fused_forward renders it,
    splatB(_rgbd)(..., moments_only=True, absgrad=True)"""
    o = ops()
    s, a = P["scales"], P["alphas"]
    if f3 is not None:
        s, a = o.filter3d_apply(s, a, f3)
    Rcw, tcw, twc = pose if pose is not None else (t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]))
    pre = o.preprocess(P["pws"], P["rots"], s, P["shs"], Rcw, tcw, twc, sc["fx"], sc["fy"], sc["cx"], sc["cy"], W, H,
                       alphas=a, antialiased=aa)
    us, ci, col, d, ar, rec = pre[:6]
    drawn = pre[6] if aa else a
    if rgbd:
        out = o.splat_rgbd(H, W, us, ci, drawn, d, col, ar, records=rec)
        return o.splatB_rgbd(H, W, us, ci, drawn, d, col, *out[1:5], *grads, moments_only=True, records=rec,
                             absgrad=True)[2]
    out = o.splat(H, W, us, ci, drawn, d, col, ar, records=rec)
    return o.splatB(H, W, us, ci, drawn, d, col, *out[1:5], grads[0], moments_only=True, records=rec, absgrad=True)[1]


@pytest.mark.parametrize("kind", ["fused", "rgbd", "pose", "rgbd_pose"])
@pytest.mark.parametrize("aa,filt", [(False, False), (True, False), (False, True), (True, True)])
def test_classes_us_abs(kind, aa, filt):
    from easygaussiansplatting_b200 import gsfunction as G
    sc, P, W, H = _class_frame()
    N = P["pws"].shape[0]
    cam = G.Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]),
                   antialiased=aa)
    f3 = torch.rand(N, device=DEV) * 0.02 if filt else None
    rgbd, posed = kind in ("rgbd", "rgbd_pose"), kind in ("pose", "rgbd_pose")
    cls = {"fused": G.GSFunctionFused, "rgbd": G.GSFunctionFusedRGBD, "pose": G.GSFunctionFusedPose,
           "rgbd_pose": G.GSFunctionFusedRGBDPose}[kind]
    rng = np.random.default_rng(3)
    gimg = t(rng.normal(size=(3, H, W)).astype(np.float32) / (3 * W * H))
    gdep, galp = t(rng.normal(size=(H, W)).astype(np.float32) / (W * H)), t(rng.normal(size=(H, W)).astype(np.float32) / (W * H))

    def run(us_abs, map_grads=True, cam_grad=posed):
        leaves = {k: v.clone().requires_grad_(map_grads) for k, v in P.items()}
        us = torch.zeros((N, 2), device=DEV, requires_grad=map_grads)
        args = [leaves["pws"], leaves["shs"], leaves["alphas"], leaves["scales"], leaves["rots"], us]
        pose = None
        if posed:
            pose = [t(sc[k]).requires_grad_(cam_grad) for k in ("Rcw", "tcw", "twc")]
            args += pose
        outs = cls.apply(*args, cam, f3, us_abs)
        loss = (outs[0] * gimg).sum()
        if rgbd:
            loss = loss + (outs[1] * gdep).sum() + (outs[2] * galp).sum()
        loss.backward()
        g = {k: v.grad for k, v in leaves.items()}
        g["us"] = us.grad
        if posed:
            g.update({k: p.grad for k, p in zip(("Rcw", "tcw", "twc"), pose)})
        return g, pose

    base, _ = run(None)
    n_abs = launches("draw_backward_rgbd_abs" if rgbd else "draw_backward_abs")
    us_abs = torch.zeros((N, 2), device=DEV, requires_grad=True)
    got, pose = run(us_abs)
    assert launches("draw_backward_rgbd_abs" if rgbd else "draw_backward_abs") == n_abs + 1
    for k, v in base.items():
        close(got[k], v, "%s with us_abs" % k, rel=1e-4)
    grads = (gimg, gdep, galp) if rgbd else (gimg,)
    want = _ops_absgrad(sc, P, W, H, aa, f3, rgbd, [p.detach() for p in pose] if posed else None, grads)
    assert us_abs.grad is not None and us_abs.grad.shape == (N, 2)
    assert float(us_abs.grad.max()) > 0
    close(us_abs.grad, want, "us_abs.grad vs the operators")
    # us_abs given without requires_grad: the plain kernel, the same gradients
    n_abs = launches("draw_backward_rgbd_abs" if rgbd else "draw_backward_abs")
    quiet = torch.zeros((N, 2), device=DEV)
    plain, _ = run(quiet)
    assert launches("draw_backward_rgbd_abs" if rgbd else "draw_backward_abs") == n_abs and quiet.grad is None
    for k, v in base.items():
        close(plain[k], v, "%s with a quiet us_abs" % k, rel=1e-4)
    if posed:  # pose only (a frozen map) with us_abs: the camera gradient and the statistic
        us_abs2 = torch.zeros((N, 2), device=DEV, requires_grad=True)
        only, _ = run(us_abs2, map_grads=False)
        for k in ("Rcw", "tcw", "twc"):
            close(only[k], base[k], "pose-only " + k, rel=1e-4)
        assert only["pws"] is None and only["us"] is None
        close(us_abs2.grad, want, "pose-only us_abs.grad")


def test_us_abs_refusals():
    from easygaussiansplatting_b200 import gsfunction as G
    sc, P, W, H = _class_frame(N=500, W=64, H=48)
    N = P["pws"].shape[0]
    cam = G.Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]))
    args = [P["pws"], P["shs"], P["alphas"], P["scales"], P["rots"], torch.zeros((N, 2), device=DEV)]
    for bad in (torch.zeros((N, 3), device=DEV), torch.zeros((N - 1, 2), device=DEV), torch.zeros(2 * N, device=DEV),
                torch.zeros((N, 2))):
        with pytest.raises(ValueError, match="us_abs"):
            G.GSFunctionFused.apply(*args, cam, None, bad.requires_grad_())
    cam.grad_exchange = object()
    with pytest.raises(ValueError, match="grad_exchange"):
        G.GSFunctionFused.apply(*args, cam, None, torch.zeros((N, 2), device=DEV, requires_grad=True))


# ---------------------------------------------------------------- 4. density control
def test_density_controller_on_the_absolute_statistic():
    from easygaussiansplatting_b200.density import DensityController, raw_thresholds
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused
    sc, P, W, H = _class_frame(N=8000, W=200, H=150, seed=4)
    N = P["pws"].shape[0]
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]))
    ctl = DensityController(2.0, verbose=False, grad_threshold=1.6e-6)
    assert ctl.grad_threshold == 1.6e-6 and ctl.th == raw_thresholds(2.0, 0.005, 1.6e-6)
    assert DensityController(2.0).th == raw_thresholds(2.0)
    acc = cnt = None
    for step in range(3):
        us = torch.zeros((N, 2), device=DEV, requires_grad=True)
        us_abs = torch.zeros((N, 2), device=DEV, requires_grad=True)
        img, mask = GSFunctionFused.apply(P["pws"], P["shs"], P["alphas"], P["scales"], P["rots"], us, cam, None,
                                          us_abs)
        (img * t(upstream_gradient(W, H, step))).sum().backward()
        assert bool((torch.linalg.norm(us_abs.grad, dim=1) >= torch.linalg.norm(us.grad, dim=1) * (1 - 1e-4)
                     - 1e-12).all())
        ctl.update_density_info(us_abs.grad, mask)
        acc, cnt = do.accumulate(n(us_abs.grad), n(mask), acc, cnt)
        assert np.array_equal(n(ctl.cunt), cnt)
        np.testing.assert_allclose(n(ctl.grad_accum), acc, rtol=1e-6, atol=0)


def test_training_with_absgrad_densification():
    """a short run toward a rendered target from blurred, too-few Gaussians: densifying on
    us_abs.grad grows the model and the loss keeps falling"""
    from easygaussiansplatting_b200.density import DensityController
    from easygaussiansplatting_b200.gau_io import adam_groups
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused
    W, H, N = 160, 120, 3000
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=60)
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]))
    with torch.no_grad():
        target, _ = GSFunctionFused.apply(t(sc["pws"]), t(sc["shs"]), t(sc["alphas"][:, None]), t(sc["scales"]),
                                          t(sc["rots"]), torch.zeros((N, 2), device=DEV), cam)
    keep = np.arange(0, N, 3)
    raw = dict(pws=sc["pws"][keep], low_shs=np.zeros((len(keep), 3)), high_shs=np.zeros((len(keep), 45)),
               alphas_raw=np.zeros((len(keep), 1)), scales_raw=np.log(sc["scales"][keep]) + 0.3,
               rots_raw=sc["rots"][keep])
    params = {k: torch.nn.Parameter(t(np.ascontiguousarray(v, np.float32))) for k, v in raw.items()}
    groups = adam_groups(params)
    for g in groups:
        g["lr"] = dict(pws=1.6e-4, low_shs=0.02).get(g["name"], g["lr"])
    opt = torch.optim.Adam(groups, lr=1e-3, eps=1e-15)
    sense = float(np.abs(sc["pws"]).max())
    ctl = None
    losses, sizes = [], []
    for step in range(90):
        Pm = params
        M = Pm["pws"].shape[0]
        us = torch.zeros((M, 2), device=DEV, requires_grad=True)
        us_abs = torch.zeros((M, 2), device=DEV, requires_grad=True)
        shs = torch.cat([Pm["low_shs"], Pm["high_shs"][:, :9]], dim=1)
        img, mask = GSFunctionFused.apply(Pm["pws"], shs, torch.sigmoid(Pm["alphas_raw"]), torch.exp(Pm["scales_raw"]),
                                          torch.nn.functional.normalize(Pm["rots_raw"], dim=1), us, cam, None, us_abs)
        loss = (img - target).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        if ctl is None:
            # no absgrad threshold has been measured for this library: take one that a fifth of the
            # first frame's visible Gaussians reach
            stat = torch.linalg.norm(us_abs.grad, dim=1)[mask]
            ctl = DensityController(sense, verbose=False, grad_threshold=float(torch.quantile(stat, 0.8)))
        ctl.update_density_info(us_abs.grad, mask)
        if step in (30, 60):
            rep = ctl.update_gaussian_density(params, opt, generator=torch.Generator(device=DEV).manual_seed(step))
            assert rep["cloned"] + rep["splited"] > 0, rep
        losses.append(float(loss.detach()))
        sizes.append(params["pws"].shape[0])
    assert np.isfinite(losses).all()
    assert sizes[-1] > sizes[0], (sizes[0], sizes[-1])
    assert np.mean(losses[-5:]) < 0.8 * np.mean(losses[:5]), losses[::10]
