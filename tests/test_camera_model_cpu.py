"""CPU checks of the camera models (pinhole, ortho, fisheye): the fp64 oracle's u, J and dJ/dpc
(oracle/camera_model_oracle.py) against central differences, on and near the axis and near the fisheye's
validity cull; the fisheye mean against an independent unprojection; ortho as the limit of a pulled-back
pinhole; the host build of the fused forward and backward's model forms (pg_fused_math.h through
tests/host_shim/camera_model_host.cpp) against the oracle; the ABI and the host-side refusals."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from easygaussiansplatting_b200.scene import COLMAP_LIKE_FISHEYE_K, camera_model_scene
from oracle import camera_model_oracle as ocm
from oracle import oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "host_shim", "_build", "libcamera_model_host.so")
W, H = 320, 240
MODEL_ID = {"pinhole": 0, "ortho": 1, "fisheye": 2}
K_WIDE = (0.05, -0.01, 0.002, -0.0005)
# a lens whose theta_d stops increasing inside the frame: theta_d' = 1 - 0.9 theta^2 + ... <= 0 near 62 degrees
K_FOLD = (-0.3, 0.0, 0.0, 0.0)
CASES = [("pinhole", None), ("ortho", None), ("fisheye", None), ("fisheye", K_WIDE), ("fisheye", (0.2, 0.05, -0.01, 0.003))]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def cm_shim():
    src = os.path.join(HERE, "host_shim", "camera_model_host.cpp")
    hdr = os.path.join(HERE, "..", "easygaussiansplatting_b200", "csrc", "pg_fused_math.h")
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", SO, src], check=True)
    return C.CDLL(SO)


def _points(rng, n):
    """camera-frame points: general, on the axis, near it (r = 1e-8 z), at the series switch and wide"""
    z = rng.uniform(0.5, 6.0, n)
    th = rng.uniform(0.0, 1.45, n)
    ph = rng.uniform(-np.pi, np.pi, n)
    pc = np.stack([z * np.tan(th) * np.cos(ph), z * np.tan(th) * np.sin(ph), z], axis=1)
    pc[0] = (0.0, 0.0, 2.0)
    pc[1] = (1e-8 * 3.0, 0.0, 3.0)
    pc[2] = (0.0, -1e-8 * 1.5, 1.5)
    pc[3] = (0.03 * 2.0 * 0.6, 0.03 * 2.0 * 0.8, 2.0)     # t = 0.03 (the fp32 kernel's switch)
    pc[4] = (1.0001e-3 * 0.8, 1.0001e-3 * 0.6, 1.0)       # just above the oracle's switch
    pc[5] = (0.9999e-3 * 0.8, 0.9999e-3 * 0.6, 1.0)       # just below it
    return pc


@pytest.mark.parametrize("model,k", CASES)
def test_oracle_against_central_differences(model, k):
    rng = np.random.default_rng(3)
    pc = _points(rng, 64)
    fx, fy, cx, cy = 300.0, 280.0, 160.0, 120.0
    u, J, dJ, valid = ocm.project(pc, model, fx, fy, cx, cy, k)
    assert valid.all()
    for c in range(3):
        h = 1e-6 * np.maximum(1.0, np.abs(pc[:, c]))
        e = np.zeros_like(pc); e[:, c] = h
        up, Jp, _, _ = ocm.project(pc + e, model, fx, fy, cx, cy, k)
        um, Jm, _, _ = ocm.project(pc - e, model, fx, fy, cx, cy, k)
        fdu = (up - um) / (2 * h[:, None])
        fdJ = (Jp - Jm) / (2 * h[:, None, None])
        scale_u = np.abs(J).max(axis=(1, 2))[:, None]
        np.testing.assert_allclose(J[:, :, c], fdu, rtol=0, atol=1e-6 * scale_u.max())
        scale_J = np.abs(dJ).max()
        np.testing.assert_allclose(dJ[:, :, :, c], fdJ, rtol=0, atol=2e-6 * scale_J)


@pytest.mark.parametrize("k", [None, K_WIDE])
def test_fisheye_on_axis_is_pinhole_jacobian(k):
    """on the axis J is the pinhole J: s -> 1/z, g -> 2 (k1 - 1/3) / z^3, h -> 1/z^2"""
    z = 2.5
    for pc in ((0.0, 0.0, z), (1e-8 * z, 0.0, z)):
        _, J, _, _ = ocm.project(np.array([pc]), "fisheye", 300.0, 280.0, 0.0, 0.0, k)
        _, Jp, _, _ = ocm.project(np.array([pc]), "pinhole", 300.0, 280.0, 0.0, 0.0)
        np.testing.assert_allclose(J, Jp, rtol=0, atol=1e-12)
        T = ocm.fisheye_terms(np.array([pc]), k)
        k1 = 0.0 if k is None else k[0]
        np.testing.assert_allclose(T["g"], 2 * (k1 - 1 / 3) / z ** 3, rtol=1e-12)


def test_fisheye_near_validity_cull():
    """K_FOLD's theta_d' crosses 0 near theta = 62 degrees: derivatives stay exact up to it, and it culls"""
    th0 = np.sqrt(1 / 0.9)  # theta_d' = 1 - 0.9 theta^2 = 0
    z = 2.0
    ths = np.array([th0 - 0.02, th0 - 0.005, th0 + 0.005, th0 + 0.1])
    pc = np.stack([z * np.tan(ths), np.zeros(4), np.full(4, z)], axis=1)
    u, J, dJ, valid = ocm.project(pc, "fisheye", 200.0, 200.0, 0.0, 0.0, K_FOLD)
    assert valid.tolist() == [True, True, False, False]
    h = 1e-7
    for c in range(3):
        e = np.zeros_like(pc); e[:, c] = h
        up, Jp = ocm.project(pc + e, "fisheye", 200.0, 200.0, 0.0, 0.0, K_FOLD)[:2]
        um, Jm = ocm.project(pc - e, "fisheye", 200.0, 200.0, 0.0, 0.0, K_FOLD)[:2]
        np.testing.assert_allclose(J[:2, :, c], ((up - um) / (2 * h))[:2], rtol=0, atol=1e-5 * np.abs(J).max())
        np.testing.assert_allclose(dJ[:2, :, :, c], ((Jp - Jm) / (2 * h))[:2], rtol=0, atol=1e-5 * np.abs(dJ).max())


@pytest.mark.parametrize("k", [None, K_WIDE, COLMAP_LIKE_FISHEYE_K])
def test_fisheye_mean_unprojects_to_the_ray(k):
    rng = np.random.default_rng(5)
    pc = _points(rng, 200)
    u = ocm.project(pc, "fisheye", 250.0, 250.0, 320.0, 240.0, k)[0]
    d = ocm.unproject_fisheye(u, 250.0, 250.0, 320.0, 240.0, k)
    np.testing.assert_allclose(d, pc / np.linalg.norm(pc, axis=1, keepdims=True), rtol=0, atol=1e-10)


def test_ortho_is_the_limit_of_a_pulled_back_pinhole():
    rng = np.random.default_rng(7)
    pc = _points(rng, 50)
    pc[:, 2] = rng.uniform(-3.0, 3.0, 50)
    f = 40.0
    uo, Jo, _, _ = ocm.project(pc, "ortho", f, f, 10.0, 20.0)
    errs = []
    for D in (1e2, 1e3, 1e4):
        up, Jp, _, _ = ocm.project(pc + np.array([0.0, 0.0, D]), "pinhole", f * D, f * D, 10.0, 20.0)
        errs.append((np.abs(up - uo).max(), np.abs(Jp - Jo).max()))
    for a, b in zip(errs, errs[1:]):  # O(1/D): tenfold D, a tenth of the error
        assert 0.08 < b[0] / a[0] < 0.12 and 0.08 < b[1] / a[1] < 0.12


def _scene(model, k, k3, seed, n=1500):
    sc = camera_model_scene(n, W, H, model, k, sh_dim=3 * k3, seed=seed)
    rng = np.random.default_rng(seed + 11)
    a, b = 0.15, -0.1  # a general camera, so that Rcw takes part in the chain
    Ry = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    Rx = np.array([[1, 0, 0], [0, np.cos(b), -np.sin(b)], [0, np.sin(b), np.cos(b)]])
    R = Ry @ Rx
    t = np.array([0.2, -0.1, 0.3])
    pc = sc["pws"].astype(np.float64)
    sc["pws"] = np.ascontiguousarray((pc - t) @ R, np.float32)  # pc = R pw + t stays the generated point
    sc["Rcw"], sc["tcw"] = R.astype(np.float32), t.astype(np.float32)
    sc["twc"] = (-(R.T @ t)).astype(np.float32)
    sc["rots"] = (sc["rots"] * rng.uniform(0.7, 1.4, (n, 1))).astype(np.float32)
    sc["pws"][rng.choice(n, n // 40, replace=False), 2] = -50.0  # behind the camera
    return sc


def _host_fwd(shim, sc, k3, model, k):
    N = len(sc["pws"])
    us = np.empty((N, 2), np.float32); ci = np.empty((N, 3), np.float32); col = np.empty((N, 3), np.float32)
    d = np.empty(N, np.float32); ar = np.empty((N, 2), np.int32); rho = np.empty(N, np.float32)
    kk = np.asarray(k if k is not None else (0, 0, 0, 0), np.float32)
    rc = shim.camera_model_forward_host(N, k3, _p(sc["pws"]), _p(sc["rots"]), _p(sc["scales"]), _p(sc["shs"]),
                                        _p(sc["Rcw"]), _p(sc["tcw"]), _p(sc["twc"]), C.c_float(sc["fx"]),
                                        C.c_float(sc["fy"]), C.c_float(sc["cx"]), C.c_float(sc["cy"]), C.c_float(W),
                                        C.c_float(H), _p(us), _p(ci), _p(col), _p(d), _p(ar), _p(rho),
                                        MODEL_ID[model], _p(kk))
    assert rc == 0
    return us, ci, col, d, ar, rho


def _stages(sc, model, k):
    return ocm.stages(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                      sc["fy"], sc["cx"], sc["cy"], W, H, model=model, k=k)


def _rel(got, ref, rows):
    ref = np.asarray(ref, np.float64).reshape(len(rows), -1)[rows]
    got = np.asarray(got, np.float64).reshape(len(rows), -1)[rows]
    return np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30)


@pytest.mark.parametrize("model,k", [c for c in CASES if c[0] != "pinhole"])
@pytest.mark.parametrize("k3", [1, 4, 16])
def test_host_forward_against_oracle(cm_shim, model, k, k3):
    sc = _scene(model, k, k3, seed=k3)
    us, ci, col, d, ar, rho = _host_fwd(cm_shim, sc, k3, model, k)
    st = _stages(sc, model, k)
    keep = st["keep"]
    assert np.array_equal(d >= 0.2, keep)
    assert (d[~keep] == -1).all() and (ar[~keep] == 0).all() and (rho[~keep] == 1).all()
    np.testing.assert_allclose(d[keep], st["pcs"][keep, 2], rtol=1e-6, atol=0)
    assert _rel(us, st["us"], keep) < 1e-6
    assert _rel(col, st["col"], np.ones(len(d), bool)) < 1e-6
    thin = ocm.oaa.thin(sc["scales"])
    ok = keep & ~thin
    assert _rel(ci, st["ci"], ok) < 1e-4
    assert np.abs(ar[ok] - st["areas"][ok]).max() <= 1
    s = ocm.oaa.scale(st["c2"], keep)
    ok2 = ok & ~ocm.oaa.flagged(sc["scales"], s)
    np.testing.assert_allclose(rho[ok2], s["rho"][ok2], rtol=1e-3, atol=0)


def test_host_fisheye_validity_cull(cm_shim):
    sc = _scene("fisheye", K_FOLD, 1, seed=2)
    d = _host_fwd(cm_shim, sc, 1, "fisheye", K_FOLD)[3]
    st = _stages(sc, "fisheye", K_FOLD)
    pc = sc["pws"].astype(np.float64) @ sc["Rcw"].T.astype(np.float64) + sc["tcw"]
    folded = (pc[:, 2] >= 0.2) & (ocm.fisheye_terms(pc, K_FOLD)["P1"] <= 0)
    assert folded.sum() > 50
    assert (d[folded] == -1).all() and (~st["keep"][folded]).all()
    sure = np.abs(ocm.fisheye_terms(pc, K_FOLD)["P1"]) > 1e-4
    assert np.array_equal((d >= 0.2)[sure], st["keep"][sure])


@pytest.mark.parametrize("model,k", [c for c in CASES if c[0] != "pinhole"])
@pytest.mark.parametrize("k3", [1, 16])
@pytest.mark.parametrize("aa", [False, True])
def test_host_backward_against_oracle(cm_shim, model, k, k3, aa):
    sc = _scene(model, k, k3, seed=10 + k3)
    N = len(sc["pws"])
    st = _stages(sc, model, k)
    rng = np.random.default_rng(k3 + 3)
    gu = rng.normal(size=(N, 2)).astype(np.float32)
    gci = (rng.normal(size=(N, 3)) * 10).astype(np.float32)
    gcol = rng.normal(size=(N, 3)).astype(np.float32)
    gz = rng.normal(size=N).astype(np.float32)
    ga = rng.normal(size=N).astype(np.float32) if aa else np.zeros(N, np.float32)
    alphas = sc["alphas"]
    kk = np.asarray(k if k is not None else (0, 0, 0, 0), np.float32)
    outs = {}
    for pose in (False, True):
        gpw = np.empty((N, 3), np.float32); gsh = np.empty((N, 3 * k3), np.float32)
        gs = np.empty((N, 3), np.float32); gq = np.empty((N, 4), np.float32); gal = np.empty(N, np.float32)
        gcam = np.zeros((N, 15), np.float32) if pose else None
        rc = cm_shim.camera_model_backward_host(
            N, k3, _p(sc["pws"]), _p(sc["rots"]), _p(sc["scales"]), _p(sc["shs"]), _p(sc["Rcw"]), _p(sc["tcw"]),
            _p(sc["twc"]), C.c_float(sc["fx"]), C.c_float(sc["fy"]), C.c_float(sc["cx"]), C.c_float(sc["cy"]),
            C.c_float(W), C.c_float(H), _p(gu), _p(gci), _p(gcol), _p(gz), _p(ga), _p(alphas), _p(gpw), _p(gsh),
            _p(gs), _p(gq), _p(gal), _p(gcam) if pose else None, int(aa), MODEL_ID[model], _p(kk))
        assert rc == 0
        outs[pose] = (gpw, gsh, gs, gq, gal, gcam)
    # the per-Gaussian gradients do not depend on the POSE form
    for a, b in zip(outs[False][:5], outs[True][:5]):
        np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-6 * max(np.abs(a).max(), 1e-30))
    gpw, gsh, gs, gq, gal, gcam = outs[True]
    Rcw = sc["Rcw"]
    ch = orc.chain_backward(Rcw, gu.reshape(N, 1, 2), gci.reshape(N, 1, 3), ga.reshape(N, 1, 1),
                            gcol.reshape(N, 1, 3), *st["J"])
    ref = {k_: ch[k_] for k_ in ("pws", "scales", "rots", "shs")}
    ref["pws"] = ref["pws"] + ocm.ordb.chain_depth(Rcw, gz.reshape(N, 1, 1), st["depths"])
    per = ocm.camera_grad(st, sc["pws"], Rcw, sc["fx"], sc["fy"], W, H, gu, gci, gcol, gz, model=model)["per"]
    if aa:
        gc2 = ocm.oaa.dcov2d_addend(st["c2"], st["keep"], alphas, ga)
        add = ocm.oaa.chain(st, Rcw, gc2)
        for k_ in ("pws", "scales", "rots"):
            ref[k_] = ref[k_] + add[k_]
        per = per + ocm.camera_grad(ocm.oaa._identity_conic(st), sc["pws"], Rcw, sc["fx"], sc["fy"], W, H,
                                    np.zeros((N, 2)), gc2, np.zeros((N, 3)), model=model)["per"]
    thin = ocm.oaa.thin(sc["scales"])
    rows = ~thin
    if aa:
        rows &= ~ocm.oaa.flagged(sc["scales"], ocm.oaa.scale(st["c2"], st["keep"]))
    # fp32 against fp64, per row relative to the row's own scale
    for name, got in (("pws", gpw), ("scales", gs), ("rots", gq), ("shs", gsh)):
        r = np.asarray(ref[name], np.float64).reshape(N, -1)
        e = np.abs(got.reshape(N, -1) - r).max(1) / np.maximum(np.abs(r).max(1), 1e-3 * np.abs(r[rows]).max())
        assert e[rows].max() < 2e-3, (name, e[rows].max())
    pe = np.abs(gcam - per).max(1) / np.maximum(np.abs(per).max(1), 1e-3 * np.abs(per[rows]).max())
    assert pe[rows].max() < 2e-3
    # culled rows: geometry gradients are exactly 0
    cull = ~st["keep"]
    assert (gs[cull] == 0).all() and (gq[cull] == 0).all()


def test_abi_exports_the_model_entry_points():
    so = os.path.join(HERE, "..", "easygaussiansplatting_b200", "libgsplat_b200.so")
    if not os.path.exists(so):
        pytest.skip("library not built")
    out = subprocess.run(["nm", "-D", "--defined-only", so], capture_output=True, text=True).stdout
    for sym in ("gsb_preprocess_forward_model", "gsb_preprocess_backward_model"):
        assert (" T %s\n" % sym) in out
    hdr = open(os.path.join(HERE, "..", "include", "gsplat_b200.h")).read()
    for s in ("GSB_CAMERA_PINHOLE 0", "GSB_CAMERA_ORTHO 1", "GSB_CAMERA_FISHEYE 2", "gsb_camera_model;"):
        assert s in hdr
    assert "#define GSB_ABI_VERSION 1" in hdr


def test_abi_argument_errors_without_a_device():
    """the model checks run before anything touches the device (N = 0: nothing launches)"""
    from easygaussiansplatting_b200 import _lib, ops
    try:
        lib = _lib.load()
    except Exception as e:  # pragma: no cover
        pytest.skip("library not loadable: %s" % e)
    z = [None] * 7

    def fwd(model, k, fx=100.0):
        cm = ops._CameraModel(model, (C.c_float * 4)(*k))
        return lib.gsb_preprocess_forward_model(0, 1, *z, fx, 100.0, 0.0, 0.0, 10.0, 10.0, *([None] * 8),
                                                C.pointer(cm), None)

    assert fwd(1, (0, 0, 0, 0)) == 0 and fwd(2, (0.1, 0, 0, 0)) == 0 and fwd(0, (0, 0, 0, 0)) == 0
    for bad in ((3, (0, 0, 0, 0), 100.0), (2, (float("nan"), 0, 0, 0), 100.0), (1, (0.1, 0, 0, 0), 100.0),
                (0, (0, 0.1, 0, 0), 100.0), (2, (0, 0, 0, 0), 0.0), (1, (0, 0, 0, 0), -5.0)):
        assert fwd(bad[0], bad[1], bad[2]) == -1
    msg = lib.gsb_last_error()
    assert b"fx and fy" in (msg if isinstance(msg, bytes) else C.string_at(msg))
    cm = ops._CameraModel(7, (C.c_float * 4)(0, 0, 0, 0))
    rc = lib.gsb_preprocess_backward_model(0, 1, *z, 100.0, 100.0, 0.0, 0.0, 10.0, 10.0, *([None] * 15), 0,
                                           C.pointer(cm), None)
    assert rc == -1


def test_python_validation_and_refusals_without_a_device():
    from easygaussiansplatting_b200 import ops
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunction
    from easygaussiansplatting_b200.parallel import GradExchange
    R, t = torch.eye(3), torch.zeros(3)
    with pytest.raises(ValueError, match="camera_model"):
        Camera(8, 8, 5, 5, 4, 4, R, t, camera_model="equirect")
    with pytest.raises(ValueError, match="fisheye"):
        Camera(8, 8, 5, 5, 4, 4, R, t, camera_model="ortho", radial_coeffs=(0.1, 0, 0, 0))
    with pytest.raises(ValueError, match="fisheye"):
        Camera(8, 8, 5, 5, 4, 4, R, t, radial_coeffs=(0, 0, 0, 0))
    with pytest.raises(ValueError, match="finite"):
        Camera(8, 8, 5, 5, 4, 4, R, t, camera_model="fisheye", radial_coeffs=(0.1, float("inf"), 0, 0))
    with pytest.raises(ValueError, match="finite"):
        Camera(8, 8, 5, 5, 4, 4, R, t, camera_model="fisheye", radial_coeffs=(0.1, 0, 0))
    with pytest.raises(ValueError, match="fx, fy"):
        Camera(8, 8, -5, 5, 4, 4, R, t, camera_model="ortho")
    cam = Camera(8, 8, 5, 5, 4, 4, R, t, camera_model="fisheye", radial_coeffs=(0.1, 0, 0, 0))
    assert cam.camera_model == "fisheye" and cam.radial_coeffs == (0.1, 0.0, 0.0, 0.0)
    assert Camera(8, 8, 5, 5, 4, 4, R, t).camera_model == "pinhole"
    # the refusals: the 7-op surface, the exchange, the 3D filter's camera table
    x = torch.zeros((4, 3))
    with pytest.raises(ValueError, match="pinhole"):
        GSFunction.apply(x, torch.zeros((4, 3)), torch.zeros((4, 1)), x, torch.zeros((4, 4)), torch.zeros((4, 2)),
                         cam)
    ex = GradExchange.__new__(GradExchange)
    with pytest.raises(ValueError, match="pinhole"):
        ex.push(x, torch.zeros((4, 4)), x, x, cam)
    with pytest.raises(ValueError, match="pinhole"):
        ops.camera_table([cam])
    with pytest.raises(ValueError, match="pinhole"):
        ops.filter3d(x.cuda(), [cam]) if torch.cuda.is_available() else ops.camera_table([Camera(8, 8, 5, 5, 4, 4, R, t),
                                                                                   cam])
    # ops: unknown model, coefficients without the fisheye, and a non-pinhole preprocessB without moment rows
    with pytest.raises(ValueError, match="camera_model"):
        ops.preprocess(x, None, None, None, None, None, None, 1, 1, 0, 0, 8, 8, camera_model="cylinder")
    with pytest.raises(ValueError, match="fisheye"):
        ops.preprocess(x, None, None, None, None, None, None, 1, 1, 0, 0, 8, 8, radial_coeffs=(0, 0, 0, 0))
    with pytest.raises(ValueError, match="moment rows"):
        ops.preprocessB(x, None, None, None, None, None, None, 1, 1, 0, 0, 8, 8, None, None, None,
                        camera_model="ortho")
    with pytest.raises(ValueError, match="focal"):
        ops.preprocess(x, None, None, None, None, None, None, 0, 1, 0, 0, 8, 8, camera_model="ortho")
