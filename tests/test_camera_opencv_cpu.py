"""CPU checks of the OpenCV radial-tangential camera model (DESIGN 3.19): the fp64 oracle's u, J and dJ/dpc
(oracle/opencv_oracle.py) against central differences, clamped and unclamped; rho_valid and the clamp limits;
zero coefficients against the pinhole oracle; the scene's unprojection; the host build of the kernels' OPENCV
forms (pg_fused_math.h through tests/host_shim/camera_opencv_host.cpp) against the oracle; the C ABI's
refusals and the new kernels' resources; the Python validation and the COLMAP camera map."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from easygaussiansplatting_b200.scene import COLMAP_LIKE_OPENCV, camera_model_scene, synthetic_scene
from oracle import camera_model_oracle as ocm
from oracle import opencv_oracle as ocv
from oracle import oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "host_shim", "_build", "libcamera_opencv_host.so")
W, H = 320, 240
COLMAP_K = COLMAP_LIKE_OPENCV[0] + COLMAP_LIKE_OPENCV[1]
SIMPLE_RADIAL_K = (0.08, 0.0, 0.0, 0.0)
BARREL_K = (-0.45, 0.05, 0.0, 0.0)          # rho_valid = 0.886: folds inside a 60-degree frame's corners
PINCUSHION_K = (0.15, 0.02, 0.0, 0.0)
TANGENTIAL_K = (0.0, 0.0, 2e-3, -1.5e-3)
KSETS = [(0.0, 0.0, 0.0, 0.0), COLMAP_K, BARREL_K, PINCUSHION_K, TANGENTIAL_K, SIMPLE_RADIAL_K]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def cv_shim():
    src = os.path.join(HERE, "host_shim", "camera_opencv_host.cpp")
    hdr = os.path.join(HERE, "..", "easygaussiansplatting_b200", "csrc", "pg_fused_math.h")
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", SO, src], check=True)
    return C.CDLL(SO)


def _points(rng, n, k, amax=0.7):
    """camera-frame points with (x/z, y/z) inside the lens's valid region (rho <= 0.97 rho_valid), the axis
    and points at 0.97 rho_valid"""
    rv = ocv.opencv_rho_valid(k[0], k[1])
    rmax = min(amax, math.sqrt(0.97 * rv)) if np.isfinite(rv) else amax
    z = rng.uniform(0.5, 6.0, n)
    r = rmax * np.sqrt(rng.uniform(0, 1, n))
    ph = rng.uniform(-np.pi, np.pi, n)
    a, b = r * np.cos(ph), r * np.sin(ph)
    a[0] = b[0] = 0.0                               # on the axis
    a[1], b[1] = 1e-7, -2e-7
    if np.isfinite(rv):
        a[2:6] = rmax * np.cos(ph[2:6])
        b[2:6] = rmax * np.sin(ph[2:6])
    pc = np.stack([a * z, b * z, z], axis=1)
    ok = ocv.opencv_valid(pc, k)[0]
    return pc[ok]


@pytest.mark.parametrize("k", KSETS)
@pytest.mark.parametrize("lim", [(10.0, 10.0), (0.4, 10.0), (10.0, 0.3), (0.4, 0.3)],
                         ids=["unclamped", "clamp_x", "clamp_y", "clamp_xy"])
def test_oracle_against_central_differences(k, lim):
    rng = np.random.default_rng(3)
    pc = _points(rng, 96, k)
    a, b = pc[:, 0] / pc[:, 2], pc[:, 1] / pc[:, 2]
    # keep away from the clamp's kink, where a central difference straddles it
    far = (np.abs(np.abs(a) - lim[0]) > 1e-3) & (np.abs(np.abs(b) - lim[1]) > 1e-3)
    pc = pc[far]
    if lim[0] < 1:
        assert (np.abs(pc[:, 0] / pc[:, 2]) > lim[0]).sum() > 5
    if lim[1] < 1:
        assert (np.abs(pc[:, 1] / pc[:, 2]) > lim[1]).sum() > 5
    fx, fy, cx, cy = 300.0, 280.0, 160.0, 120.0
    proj = lambda q: ocv.project(q, "opencv", fx, fy, cx, cy, k, lim=lim)
    u, J, dJ, valid, Ju = proj(pc)
    assert valid.all()
    for c in range(3):
        h = 1e-6 * np.maximum(1.0, np.abs(pc[:, c]))
        e = np.zeros_like(pc); e[:, c] = h
        up, Jp = proj(pc + e)[:2]
        um, Jm = proj(pc - e)[:2]
        np.testing.assert_allclose(Ju[:, :, c], (up - um) / (2 * h[:, None]), rtol=0, atol=1e-6 * np.abs(Ju).max())
        np.testing.assert_allclose(dJ[:, :, :, c], (Jp - Jm) / (2 * h[:, None, None]), rtol=0,
                                   atol=2e-6 * np.abs(dJ).max())
    inside = (np.abs(pc[:, 0] / pc[:, 2]) <= lim[0]) & (np.abs(pc[:, 1] / pc[:, 2]) <= lim[1])
    np.testing.assert_array_equal(J[inside], Ju[inside])


def test_zero_coefficients_are_the_pinhole_projection():
    rng = np.random.default_rng(4)
    pc = _points(rng, 64, (0, 0, 0, 0))
    u, J, dJ, valid, Ju = ocv.project(pc, "opencv", 300.0, 280.0, 160.0, 120.0, None, lim=(10.0, 10.0))
    up, Jp, dJp, _ = ocm.project(pc, "pinhole", 300.0, 280.0, 160.0, 120.0)
    np.testing.assert_allclose(u, up, rtol=1e-14, atol=1e-12)
    np.testing.assert_allclose(J, Jp, rtol=1e-14, atol=1e-12)
    np.testing.assert_allclose(Ju, Jp, rtol=1e-14, atol=1e-12)
    np.testing.assert_allclose(dJ, dJp, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("k", KSETS)
def test_rho_valid_against_a_dense_scan(k):
    k1, k2 = k[:2]
    rho = np.linspace(0, 20, 2_000_001)
    d = 1 + 3 * k1 * rho + 5 * k2 * rho ** 2
    rv = ocv.opencv_rho_valid(k1, k2)
    neg = np.nonzero(d <= 0)[0]
    if len(neg) == 0:
        assert rv > 20 or not np.isfinite(rv)
    else:
        assert abs(rv - rho[neg[0]]) <= 2e-5
    for kk in ((-0.3, 0.0), (0.0, -0.1), (0.2, 0.1), (-0.6, 0.2), (0.1, -0.02)):
        d = 1 + 3 * kk[0] * rho + 5 * kk[1] * rho ** 2
        neg = np.nonzero(d <= 0)[0]
        rv = ocv.opencv_rho_valid(*kk)
        assert (not np.isfinite(rv)) if len(neg) == 0 else abs(rv - rho[neg[0]]) <= 2e-5, kk


def test_limits_are_pinhole_without_radial_terms():
    for k in ((0, 0, 0, 0), TANGENTIAL_K, None):
        assert ocv.opencv_limits(k, 300.0, 280.0, 150.0, 110.0, W, H) == (1.3 * W / 600.0, 1.3 * H / 560.0)


@pytest.mark.parametrize("k", KSETS)
def test_image_border_undistorts_inside_the_limits(k):
    """with a centred principal point every border pixel's undistorted point lies inside (Lx, Ly): the
    clamp never touches a Gaussian whose mean is on screen"""
    sc = synthetic_scene(1, W, H)
    fx, fy, cx, cy = sc["fx"], sc["fy"], sc["cx"], sc["cy"]
    Lx, Ly = ocv.opencv_limits(k, fx, fy, cx, cy, W, H)
    t = np.linspace(0, 1, 401)
    border = np.concatenate([np.stack([t * W, np.zeros_like(t)], 1), np.stack([t * W, np.full_like(t, H)], 1),
                             np.stack([np.zeros_like(t), t * H], 1), np.stack([np.full_like(t, W), t * H], 1)])
    ab = ocv.unproject_opencv(border, fx, fy, cx, cy, k)
    rv = ocv.opencv_rho_valid(k[0], k[1])
    reach = np.array([ocv._solve_radial(np.hypot((u - cx) / fx, (v - cy) / fy), k[0], k[1]) for u, v in border])
    ok = ~np.isclose(reach ** 2, rv, rtol=1e-9) if np.isfinite(rv) else np.ones(len(border), bool)
    assert ok.sum() > len(border) // 2
    assert (np.abs(ab[ok, 0]) < Lx).all() and (np.abs(ab[ok, 1]) < Ly).all()
    # the unprojection is exact where it converged
    u = ocv.project(np.c_[ab[ok], np.ones(ok.sum())], "opencv", fx, fy, cx, cy, k, lim=(Lx, Ly))[0]
    np.testing.assert_allclose(u, border[ok], rtol=0, atol=1e-8)


def _scene(k, k3, seed, n=1500, posed=True):
    sc = camera_model_scene(n, W, H, "opencv", k[:2], sh_dim=3 * k3, seed=seed, tangential_coeffs=k[2:])
    rng = np.random.default_rng(seed + 11)
    if posed:
        a, b = 0.15, -0.1
        Ry = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        Rx = np.array([[1, 0, 0], [0, np.cos(b), -np.sin(b)], [0, np.sin(b), np.cos(b)]])
        R = Ry @ Rx
        t = np.array([0.2, -0.1, 0.3])
        pc = sc["pws"].astype(np.float64)
        sc["pws"] = np.ascontiguousarray((pc - t) @ R, np.float32)
        sc["Rcw"], sc["tcw"] = R.astype(np.float32), t.astype(np.float32)
        sc["twc"] = (-(R.T @ t)).astype(np.float32)
    sc["rots"] = (sc["rots"] * rng.uniform(0.7, 1.4, (n, 1))).astype(np.float32)
    sc["pws"][rng.choice(n, n // 40, replace=False), 2] = -50.0
    return sc


def _stages(sc, k, model="opencv"):
    return ocv.stages(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                      sc["fy"], sc["cx"], sc["cy"], W, H, model=model, k=k)


@pytest.mark.parametrize("k", [COLMAP_K, BARREL_K])
def test_scene_unprojection_round_trips(k):
    sc = camera_model_scene(400, W, H, "opencv", k[:2], seed=5, tangential_coeffs=k[2:])
    rng = np.random.default_rng(5)  # synthetic_scene's draws
    z = rng.uniform(2.0, 12.0, 400)
    u = rng.uniform(-0.05 * W, 1.05 * W, 400)
    v = rng.uniform(-0.05 * H, 1.05 * H, 400)
    pc = sc["pws"].astype(np.float64)
    np.testing.assert_allclose(pc[:, 2], z, rtol=1e-6)
    got, _, _, valid, _ = ocv.project(pc, "opencv", sc["fx"], sc["fy"], sc["cx"], sc["cy"], k, lim=(10.0, 10.0))
    assert valid.sum() > 300
    np.testing.assert_allclose(got[valid], np.stack([u, v], 1)[valid], rtol=0, atol=2e-3)  # float32 positions
    if k == BARREL_K:
        assert (~valid).sum() > 5  # corner targets beyond the fold are placed past it


def test_zero_coefficients_against_pinhole_stages():
    """the forward everywhere; the backward (du/dpc always, dcov2d/dpc where nothing is clamped: pinhole keeps
    the reference's unclamped-x, y derivative on clamped rows)"""
    sc = _scene((0, 0, 0, 0), 4, seed=1, posed=False)
    wide = np.arange(0, 1500, 10)  # beyond the clamp in x, y or both
    sc["pws"][wide, 0] *= np.where(wide % 20 == 0, 1.8, 1.0) * 1.1
    sc["pws"][wide[1::3], 1] *= 2.5
    st = _stages(sc, (0, 0, 0, 0))
    sp = _stages(sc, None, model="pinhole")
    # the pinhole stages come from the fp32 C oracle: equal to its rounding
    for key in ("us", "ci", "col", "depths", "areas", "keep", "c2"):
        ref = np.asarray(sp[key], np.float64)
        np.testing.assert_allclose(np.asarray(st[key], np.float64), ref, rtol=1e-6, atol=1e-6 * np.abs(ref).max(),
                                   err_msg=key)
    pc = st["pcs"].astype(np.float64)
    lim = st["lim"]
    with np.errstate(invalid="ignore", divide="ignore"):
        unc = st["keep"] & (np.abs(pc[:, 0] / pc[:, 2]) < lim[0]) & (np.abs(pc[:, 1] / pc[:, 2]) < lim[1])
    assert (st["keep"] & ~unc).sum() > 10 and unc.sum() > 1000
    for i, (a, b) in enumerate(zip(st["J"], sp["J"])):
        a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
        rows = unc if i == 4 else np.ones(len(a), bool)
        np.testing.assert_allclose(a[rows], b[rows], rtol=1e-6, atol=1e-6 * np.abs(b).max(), err_msg=str(i))


def _host_fwd(shim, sc, k3, k, lim):
    N = len(sc["pws"])
    us = np.empty((N, 2), np.float32); ci = np.empty((N, 3), np.float32); col = np.empty((N, 3), np.float32)
    d = np.empty(N, np.float32); ar = np.empty((N, 2), np.int32); rho = np.empty(N, np.float32)
    kk = np.asarray(k, np.float32)
    rc = shim.camera_opencv_forward_host(N, k3, _p(sc["pws"]), _p(sc["rots"]), _p(sc["scales"]), _p(sc["shs"]),
                                         _p(sc["Rcw"]), _p(sc["tcw"]), _p(sc["twc"]), C.c_float(sc["fx"]),
                                         C.c_float(sc["fy"]), C.c_float(sc["cx"]), C.c_float(sc["cy"]),
                                         C.c_float(lim[0] / 1.3), C.c_float(lim[1] / 1.3), _p(us), _p(ci), _p(col),
                                         _p(d), _p(ar), _p(rho), _p(kk))
    assert rc == 0
    return us, ci, col, d, ar, rho


def _rel(got, ref, rows):
    ref = np.asarray(ref, np.float64).reshape(len(rows), -1)[rows]
    got = np.asarray(got, np.float64).reshape(len(rows), -1)[rows]
    return np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30)


def _band(sc, k):
    pc = sc["pws"].astype(np.float64) @ sc["Rcw"].T.astype(np.float64) + sc["tcw"]
    return (pc[:, 2] > 0.2) & ocv.opencv_band(pc, k, sc["fx"], sc["fy"], sc["cx"], sc["cy"], W, H)


@pytest.mark.parametrize("k", KSETS)
@pytest.mark.parametrize("k3", [1, 4, 16])
def test_host_forward_against_oracle(cv_shim, k, k3):
    sc = _scene(k, k3, seed=k3)
    st = _stages(sc, k)
    us, ci, col, d, ar, rho = _host_fwd(cv_shim, sc, k3, k, st["lim"])
    keep = st["keep"]
    sure = ~_band(sc, k)
    assert np.array_equal((d >= 0.2)[sure], keep[sure])
    keep = keep & sure & (d >= 0.2)
    assert (d[d < 0.2] == -1).all() and (ar[d < 0.2] == 0).all() and (rho[d < 0.2] == 1).all()
    np.testing.assert_allclose(d[keep], st["pcs"][keep, 2], rtol=1e-6, atol=0)
    assert _rel(us, st["us"], keep) < 1e-6
    assert _rel(col, st["col"], np.ones(len(d), bool)) < 1e-6
    thin = ocm.oaa.thin(sc["scales"])
    ok = keep & ~thin
    assert _rel(ci, st["ci"], ok) < 1e-4
    assert np.abs(ar[ok] - st["areas"][ok]).max() <= 1
    s = ocm.oaa.scale(st["c2"], st["keep"])
    ok2 = ok & ~ocm.oaa.flagged(sc["scales"], s)
    np.testing.assert_allclose(rho[ok2], s["rho"][ok2], rtol=1e-3, atol=0)


def test_host_validity_cull(cv_shim):
    """BARREL_K folds inside the frame (rho >= rho_valid); a strong tangential lens folds by det Ddelta <= 0"""
    for k, which in ((BARREL_K, 1), ((0.0, 0.0, 0.2, 0.0), 2)):
        sc = _scene(k, 1, seed=2, posed=False)
        st = _stages(sc, k)
        d = _host_fwd(cv_shim, sc, 1, k, st["lim"])[3]
        pc = sc["pws"].astype(np.float64)
        valid, drho, det = ocv.opencv_valid(pc, k)
        folded = (pc[:, 2] >= 0.2) & ~valid
        assert folded.sum() > 20, k
        assert ((drho <= 0) if which == 1 else (det <= 0))[folded].any()
        assert (d[folded] == -1).all() and (~st["keep"][folded]).all()
        sure = ~_band(sc, k)
        assert np.array_equal((d >= 0.2)[sure], st["keep"][sure])


@pytest.mark.parametrize("k", [(0.0, 0.0, 0.0, 0.0), COLMAP_K, BARREL_K, TANGENTIAL_K])
@pytest.mark.parametrize("k3", [1, 16])
@pytest.mark.parametrize("aa", [False, True])
def test_host_backward_against_oracle(cv_shim, k, k3, aa):
    sc = _scene(k, k3, seed=10 + k3)
    N = len(sc["pws"])
    st = _stages(sc, k)
    rng = np.random.default_rng(k3 + 3)
    gu = rng.normal(size=(N, 2)).astype(np.float32)
    gci = (rng.normal(size=(N, 3)) * 10).astype(np.float32)
    gcol = rng.normal(size=(N, 3)).astype(np.float32)
    gz = rng.normal(size=N).astype(np.float32)
    ga = rng.normal(size=N).astype(np.float32) if aa else np.zeros(N, np.float32)
    alphas = sc["alphas"]
    kk = np.asarray(k, np.float32)
    outs = {}
    for pose in (False, True):
        gpw = np.empty((N, 3), np.float32); gsh = np.empty((N, 3 * k3), np.float32)
        gs = np.empty((N, 3), np.float32); gq = np.empty((N, 4), np.float32); gal = np.empty(N, np.float32)
        gcam = np.zeros((N, 15), np.float32) if pose else None
        rc = cv_shim.camera_opencv_backward_host(
            N, k3, _p(sc["pws"]), _p(sc["rots"]), _p(sc["scales"]), _p(sc["shs"]), _p(sc["Rcw"]), _p(sc["tcw"]),
            _p(sc["twc"]), C.c_float(sc["fx"]), C.c_float(sc["fy"]), C.c_float(sc["cx"]), C.c_float(sc["cy"]),
            C.c_float(st["lim"][0] / 1.3), C.c_float(st["lim"][1] / 1.3), _p(gu), _p(gci), _p(gcol), _p(gz), _p(ga),
            _p(alphas), _p(gpw), _p(gsh), _p(gs), _p(gq), _p(gal), _p(gcam) if pose else None, int(aa), _p(kk))
        assert rc == 0
        outs[pose] = (gpw, gsh, gs, gq, gal, gcam)
    for a, b in zip(outs[False][:5], outs[True][:5]):
        np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-6 * max(np.abs(a).max(), 1e-30))
    gpw, gsh, gs, gq, gal, gcam = outs[True]
    Rcw = sc["Rcw"]
    ch = orc.chain_backward(Rcw, gu.reshape(N, 1, 2), gci.reshape(N, 1, 3), ga.reshape(N, 1, 1),
                            gcol.reshape(N, 1, 3), *st["J"])
    ref = {k_: ch[k_] for k_ in ("pws", "scales", "rots", "shs")}
    ref["pws"] = ref["pws"] + ocm.ordb.chain_depth(Rcw, gz.reshape(N, 1, 1), st["depths"])
    per = ocv.camera_grad(st, sc["pws"], Rcw, sc["fx"], sc["fy"], W, H, gu, gci, gcol, gz, model="opencv")["per"]
    if aa:
        gc2 = ocm.oaa.dcov2d_addend(st["c2"], st["keep"], alphas, ga)
        add = ocm.oaa.chain(st, Rcw, gc2)
        for k_ in ("pws", "scales", "rots"):
            ref[k_] = ref[k_] + add[k_]
        per = per + ocv.camera_grad(ocm.oaa._identity_conic(st), sc["pws"], Rcw, sc["fx"], sc["fy"], W, H,
                                    np.zeros((N, 2)), gc2, np.zeros((N, 3)), model="opencv")["per"]
    rows = ~ocm.oaa.thin(sc["scales"]) & ~_band(sc, k)
    if aa:
        rows &= ~ocm.oaa.flagged(sc["scales"], ocm.oaa.scale(st["c2"], st["keep"]))
    for name, got in (("pws", gpw), ("scales", gs), ("rots", gq), ("shs", gsh)):
        r = np.asarray(ref[name], np.float64).reshape(N, -1)
        e = np.abs(got.reshape(N, -1) - r).max(1) / np.maximum(np.abs(r).max(1), 1e-3 * np.abs(r[rows]).max())
        assert e[rows].max() < 2e-3, (name, e[rows].max())
    pe = np.abs(gcam - per).max(1) / np.maximum(np.abs(per).max(1), 1e-3 * np.abs(per[rows]).max())
    assert pe[rows].max() < 2e-3
    cull = ~st["keep"] & rows
    assert (gs[cull] == 0).all() and (gq[cull] == 0).all()


def test_abi_header_and_refusals_without_a_device():
    hdr = open(os.path.join(HERE, "..", "include", "gsplat_b200.h")).read()
    assert "#define GSB_CAMERA_OPENCV 4" in hdr and "#define GSB_ABI_VERSION 1" in hdr
    assert not re.search(r"#define GSB_CAMERA_\w+ 3\b", hdr)
    from easygaussiansplatting_b200 import _lib, ops
    try:
        lib = _lib.load()
    except Exception as e:  # pragma: no cover
        pytest.skip("library not loadable: %s" % e)
    z = [None] * 7

    def fwd(model, k, fx=100.0, fy=100.0, w=10.0, h=10.0):
        cm = ops._CameraModel(model, (C.c_float * 4)(*k))
        return lib.gsb_preprocess_forward_model(0, 1, *z, fx, fy, 5.0, 5.0, w, h, *([None] * 8), C.pointer(cm), None)

    def msg():
        m = lib.gsb_last_error()
        return m if isinstance(m, bytes) else C.string_at(m)

    assert fwd(4, (0, 0, 0, 0)) == 0 and fwd(4, (-0.2, 0.05, 1e-3, -1e-3)) == 0 and fwd(4, (-5.0, 0, 0, 0)) == 0
    for bad in ((float("nan"), 0, 0, 0), (0, float("inf"), 0, 0), (0, 0, 0, float("-inf"))):
        assert fwd(4, bad) == -1 and b"finite" in msg()
    assert fwd(4, (0.1, 0, 0, 0), fx=0.0) == -1 and b"fx and fy" in msg()
    assert fwd(4, (0.1, 0, 0, 0), fy=-1.0) == -1 and b"fx and fy" in msg()
    assert fwd(4, (0.1, 0, 0, 0), w=0.0) == -1 and b"width and height" in msg()
    assert fwd(4, (0.1, 0, 0, 0), h=-3.0) == -1 and b"width and height" in msg()
    for model in (0, 1):
        for k in ((0.1, 0, 0, 0), (0, 0, 0.01, 0)):
            assert fwd(model, k) == -1
    assert fwd(3, (0, 0, 0, 0)) == -1 and b"unknown" in msg()
    cm = ops._CameraModel(4, (C.c_float * 4)(0.1, 0, 0, 0))
    rc = lib.gsb_preprocess_backward_model(0, 1, *z, 100.0, 100.0, 0.0, 0.0, 0.0, 10.0, *([None] * 15), 0,
                                           C.pointer(cm), None)
    assert rc == -1 and b"width and height" in msg()


def test_opencv_kernels_are_sm90a_without_spills():
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    r = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True)
    assert r.returncode == 0
    found = {}
    for name, usage in re.findall(r"Function (_ZN3gsb16k_preprocess_(?:fwd|bwd)\S+):\s*\n\s*(REG:.*)", r.stdout):
        m = re.search(r"k_preprocess_(fwd|bwd)ILi(\d+)E((?:Lb\dE)+)Li(\d)EEEv", name)
        if m and m.group(4) == "4":
            found[(m.group(1), m.group(2), m.group(3))] = usage
    # the forward at every K3 x AA; the backward with MOM, without PUSH, at every K3 x DEPTH x POSE x AA
    want = {("fwd", k3, "Lb%sE" % a) for k3 in ("1", "4", "9", "16") for a in "01"}
    want |= {("bwd", k3, "Lb0ELb1ELb%sELb%sELb%sE" % (d, p, a)) for k3 in ("1", "4", "9", "16") for d in "01"
             for p in "01" for a in "01"}
    assert set(found) == want
    for t, usage in found.items():
        assert "STACK:0 " in usage and "LOCAL:0 " in usage, (t, usage)


def test_python_validation_without_a_device():
    from easygaussiansplatting_b200 import ops
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunction
    from easygaussiansplatting_b200.parallel import GradExchange
    R, t = torch.eye(3), torch.zeros(3)
    cam = Camera(8, 8, 5, 5, 4, 4, R, t, camera_model="opencv", radial_coeffs=(-0.1, 0.01), tangential_coeffs=(1e-3, 0))
    assert cam.camera_model == "opencv" and cam.radial_coeffs == (-0.1, 0.01) and cam.tangential_coeffs == (1e-3, 0.0)
    cam0 = Camera(8, 8, 5, 5, 4, 4, R, t, camera_model="opencv")
    assert cam0.radial_coeffs is None and cam0.tangential_coeffs is None
    assert ops.camera_model_args("opencv", (0.1, 0.2), (0.3, 0.4)) == ("opencv", (0.1, 0.2, 0.3, 0.4))
    assert ops.camera_model_args("opencv", None, (0.3, 0.4)) == ("opencv", (0.0, 0.0, 0.3, 0.4))
    assert ops._CAMERA_MODEL_ID["opencv"] == 4
    with pytest.raises(ValueError, match="finite"):
        Camera(8, 8, 5, 5, 4, 4, R, t, camera_model="opencv", radial_coeffs=(0.1, 0, 0, 0))
    with pytest.raises(ValueError, match="finite"):
        Camera(8, 8, 5, 5, 4, 4, R, t, camera_model="opencv", radial_coeffs=(0.1, float("nan")))
    with pytest.raises(ValueError, match="finite"):
        Camera(8, 8, 5, 5, 4, 4, R, t, camera_model="opencv", tangential_coeffs=(0.1,))
    with pytest.raises(ValueError, match="opencv"):
        Camera(8, 8, 5, 5, 4, 4, R, t, camera_model="fisheye", tangential_coeffs=(0.1, 0))
    with pytest.raises(ValueError, match="opencv"):
        Camera(8, 8, 5, 5, 4, 4, R, t, tangential_coeffs=(0, 0))
    with pytest.raises(ValueError, match="fx, fy"):
        Camera(8, 8, 5, 0, 4, 4, R, t, camera_model="opencv")
    with pytest.raises(ValueError, match="opencv"):
        ops.preprocess(torch.zeros((4, 3)), None, None, None, None, None, None, 1, 1, 0, 0, 8, 8,
                       tangential_coeffs=(0, 0))
    with pytest.raises(ValueError, match="moment rows"):
        ops.preprocessB(torch.zeros((4, 3)), None, None, None, None, None, None, 1, 1, 0, 0, 8, 8, None, None, None,
                        camera_model="opencv")
    with pytest.raises(ValueError, match="focal"):
        ops.preprocess(torch.zeros((4, 3)), None, None, None, None, None, None, 1, -1, 0, 0, 8, 8,
                       camera_model="opencv")
    # the pinhole-only surfaces refuse it as they refuse the fisheye
    x = torch.zeros((4, 3))
    with pytest.raises(ValueError, match="pinhole"):
        GSFunction.apply(x, torch.zeros((4, 3)), torch.zeros((4, 1)), x, torch.zeros((4, 4)), torch.zeros((4, 2)),
                         cam)
    ex = GradExchange.__new__(GradExchange)
    with pytest.raises(ValueError, match="pinhole"):
        ex.push(x, torch.zeros((4, 4)), x, x, cam)
    with pytest.raises(ValueError, match="pinhole"):
        ops.camera_table([cam])


def test_colmap_intrinsics_all_models():
    from easygaussiansplatting_b200.gsfunction import Camera, colmap_intrinsics
    R, t = torch.eye(3), torch.zeros(3)
    cases = {
        "SIMPLE_PINHOLE": ([500.0, 320.0, 240.0], dict(fx=500.0, fy=500.0, cx=320.0, cy=240.0, camera_model="pinhole",
                                                       radial_coeffs=None, tangential_coeffs=None)),
        "PINHOLE": ([500.0, 510.0, 321.0, 239.0], dict(fx=500.0, fy=510.0, cx=321.0, cy=239.0, camera_model="pinhole",
                                                       radial_coeffs=None, tangential_coeffs=None)),
        "SIMPLE_RADIAL": ([500.0, 320.0, 240.0, -0.05], dict(fx=500.0, fy=500.0, cx=320.0, cy=240.0,
                                                             camera_model="opencv", radial_coeffs=(-0.05, 0.0),
                                                             tangential_coeffs=None)),
        "RADIAL": ([500.0, 320.0, 240.0, -0.05, 0.01], dict(fx=500.0, fy=500.0, cx=320.0, cy=240.0,
                                                            camera_model="opencv", radial_coeffs=(-0.05, 0.01),
                                                            tangential_coeffs=None)),
        "OPENCV": ([500.0, 510.0, 321.0, 239.0, -0.05, 0.01, 1e-3, -2e-3],
                   dict(fx=500.0, fy=510.0, cx=321.0, cy=239.0, camera_model="opencv", radial_coeffs=(-0.05, 0.01),
                        tangential_coeffs=(1e-3, -2e-3))),
        "OPENCV_FISHEYE": ([300.0, 301.0, 320.0, 240.0, 0.05, -0.01, 0.002, -0.0005],
                           dict(fx=300.0, fy=301.0, cx=320.0, cy=240.0, camera_model="fisheye",
                                radial_coeffs=(0.05, -0.01, 0.002, -0.0005), tangential_coeffs=None)),
    }
    for name, (params, want) in cases.items():
        got = colmap_intrinsics(name, params, 640, 480)
        assert got == want, name
        Camera(640, 480, Rcw=R, tcw=t, **got)
        # a half-size image: focal lengths and principal point halve, coefficients stay
        half = colmap_intrinsics(name, np.array(params), 640, 480, image_width=320, image_height=240)
        for key in ("fx", "fy", "cx", "cy"):
            assert half[key] == want[key] / 2, (name, key)
        for key in ("camera_model", "radial_coeffs", "tangential_coeffs"):
            assert half[key] == want[key], (name, key)
        # an anisotropic resize scales x and y apart
        an = colmap_intrinsics(name, params, 640, 480, image_width=1280, image_height=240)
        assert an["fx"] == 2 * want["fx"] and an["cx"] == 2 * want["cx"]
        assert an["fy"] == want["fy"] / 2 and an["cy"] == want["cy"] / 2
        with pytest.raises(ValueError, match=name):
            colmap_intrinsics(name, params + [0.0], 640, 480)
        with pytest.raises(ValueError, match=name):
            colmap_intrinsics(name, params[:-1], 640, 480)
    for name in ("FULL_OPENCV", "FOV", "SIMPLE_RADIAL_FISHEYE", "RADIAL_FISHEYE", "THIN_PRISM_FISHEYE", "opencv"):
        with pytest.raises(ValueError, match=name):
            colmap_intrinsics(name, [1.0] * 12, 640, 480)
