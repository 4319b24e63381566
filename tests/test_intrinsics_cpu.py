"""The intrinsics gradient without a GPU (DESIGN 3.23): the fp64 oracle against central differences per
Gaussian under every camera model (clamped rows under the constant-bound rule, antialiasing's term), the
workspace queries, every argument error of the two entry points returned before any launch, the Python
argument rules, and the new kernels in the sm_90a cubin without stack or spills."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import aa_oracle as oaa
from oracle import camera_model_oracle as ocm
from oracle import intrinsics_oracle as oin
from oracle import opencv_oracle as ocv
from oracle import step_oracle as ost
from easygaussiansplatting_b200.scene import camera_model_scene

HERE = os.path.dirname(os.path.abspath(__file__))
SHIM_SO = os.path.join(HERE, "host_shim", "_build", "libintrinsics_host.so")
MODEL_ID = {"pinhole": 0, "ortho": 1, "fisheye": 2, "opencv": 4}

CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
KS = {"pinhole": (0, 0, 0, 0), "ortho": (0, 0, 0, 0), "fisheye": (0.05, -0.01, 0.004, -0.001),
      "opencv": (-0.08, 0.02, 0.001, -0.002)}


def _gaussians(N, seed, model):
    """N Gaussians in front of the camera: some near the axis (fisheye's series branch), some beyond the
    pinhole / opencv clamp bound; random covariances and a random rotation"""
    rng = np.random.default_rng(seed)
    z = rng.uniform(1.0, 4.0, N)
    tx = rng.uniform(-0.9, 0.9, N)
    tx[: N // 8] = rng.uniform(-0.02, 0.02, N // 8)                       # t < 0.03
    tx[N // 8: N // 4] = np.sign(rng.normal(size=N // 8)) * rng.uniform(0.8, 1.0, N // 8)  # past 1.3 tan_fov
    ty = rng.uniform(-0.5, 0.5, N)
    ty[: N // 8] = rng.uniform(-0.02, 0.02, N // 8)
    pc = np.stack([tx * z, ty * z, z], 1)
    A = rng.normal(size=(N, 3, 3)) * 0.08
    S = A @ A.transpose(0, 2, 1) + 0.01 * np.eye(3)
    c3 = S[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, zq = q
    R = np.array([[1 - 2 * (y * y + zq * zq), 2 * (x * y - zq * w), 2 * (x * zq + y * w)],
                  [2 * (x * y + zq * w), 1 - 2 * (x * x + zq * zq), 2 * (y * zq - x * w)],
                  [2 * (x * zq - y * w), 2 * (y * zq + x * w), 1 - 2 * (x * x + y * y)]])
    return pc, R, c3, rng


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("model", oin.MODELS)
def test_oracle_per_gaussian_vs_central_differences(model, aa):
    """L_n = gu . u + gconic . conic (+ galpha alpha rho with AA) of each Gaussian, differentiated by each of the
    8 intrinsics with the clamp bound pinned, against oin.per_gaussian"""
    W, H = 640, 480
    N = 64
    pc, R, c3, rng = _gaussians(N, 7 + MODEL_SEED[model], model)
    assert (np.hypot(pc[:, 0], pc[:, 1]) < 0.03 * pc[:, 2]).sum() >= N // 8
    intr = np.array([520.0, 500.0, 322.0, 236.0] + list(KS[model]))
    if model == "ortho":
        intr[:2] = [90.0, 85.0]
    lim = oin.limits(model, intr, W, H)
    if lim is not None:
        assert (np.abs(pc[:, 0] / pc[:, 2]) > lim[0]).any() and (np.abs(pc[:, 0] / pc[:, 2]) < lim[0]).any()
    gu = rng.normal(size=(N, 2))
    gcon = rng.normal(size=(N, 3)) * 50
    galpha = rng.normal(size=N) if aa else np.zeros(N)
    alpha = rng.uniform(0.2, 0.9, N)
    u0, ci0, rho0 = oin.forward(pc, R, c3, model, intr, lim)
    add = None
    if aa:
        c2 = oin._cov2d(oin.dproj(pc, model, intr, lim)[1], R, c3)[0]
        add = oaa.dcov2d_addend(c2, np.ones(N, bool), alpha, galpha)
        assert (rho0 ** 2 > oaa.R_MIN).all()
    an = oin.per_gaussian(pc, R, c3, model, intr, lim, gu, gcon, add)

    def loss(th):
        u, ci, rho = oin.forward(pc, R, c3, model, th, lim)
        return (gu * u).sum(1) + (gcon * ci).sum(1) + galpha * alpha * rho

    for j in range(8):
        h = 1e-6 * max(abs(intr[j]), 1.0)
        tp, tm = intr.copy(), intr.copy()
        tp[j] += h
        tm[j] -= h
        fd = (loss(tp) - loss(tm)) / (2 * h)
        scale = np.abs(an).max(1) + np.abs(gu).sum(1)
        err = np.abs(fd - an[:, j]) / scale
        assert err.max() < 1e-6, (model, aa, j, err.max())
        if model in ("pinhole", "ortho") and j >= 4:
            assert not an[:, j].any()
    assert np.abs(an[:, 4:]).max() > 0 or model in ("pinhole", "ortho")


MODEL_SEED = {m: i for i, m in enumerate(oin.MODELS)}


@pytest.fixture(scope="module")
def shim():
    """tests/host_shim/intrinsics_host.cpp: backward_one's intrinsics mode, host build"""
    src = os.path.join(HERE, "host_shim", "intrinsics_host.cpp")
    hdr = os.path.join(HERE, "..", "easygaussiansplatting_b200", "csrc", "pg_fused_math.h")
    os.makedirs(os.path.dirname(SHIM_SO), exist_ok=True)
    if not os.path.exists(SHIM_SO) or os.path.getmtime(SHIM_SO) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", SHIM_SO, src],
                       check=True)
    return C.CDLL(SHIM_SO)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


SHIM_K = {"pinhole": (0, 0, 0, 0), "ortho": (0, 0, 0, 0), "fisheye": (0.05, -0.01, 0.004, -0.001),
          "opencv": (-0.25, 0.01, 0.001, -0.002)}


def _shim_scene(model, k3, seed):
    """camera-frame points by band: near the axis (|x/z|, |y/z| < 0.015: fisheye's series branch), just past
    t = 0.03, spread over the frame, past the clamp bound (pinhole, opencv), and (opencv) between 0.9 and
    0.99 of the fold radius; random covariances, a rotated camera -> the shim's fp32 inputs and the oracle's"""
    rng = np.random.default_rng(seed)
    W, H = 640.0, 480.0
    f = 90.0 if model == "ortho" else 400.0
    intr = [f, f * 0.97, W / 2 + 5, H / 2 - 3] + list(SHIM_K[model])
    lim = oin.limits(model, intr, W, H)
    n = 48
    z = rng.uniform(1.0, 5.0, 6 * n)
    ang = rng.uniform(0, 2 * np.pi, 6 * n)
    t = np.concatenate([rng.uniform(0, 0.015, n), rng.uniform(0.031, 0.06, n), rng.uniform(0.06, 0.6, 2 * n),
                        rng.uniform(1.05, 1.4, n) * (lim[0] if lim else 0.6),
                        np.sqrt(rng.uniform(0.9, 0.99, n) * ocv.opencv_rho_valid(*SHIM_K["opencv"][:2]))
                        if model == "opencv" else rng.uniform(0.6, 1.0, n)])
    a, b = t * np.cos(ang), t * np.sin(ang)
    if model == "ortho":
        pc = np.stack([a * 2, b * 2, z], 1)
    else:
        pc = np.stack([a * z, b * z, z], 1)
    N = len(pc)
    th = 0.3
    R = np.array([[np.cos(th), 0, np.sin(th)], [0, 1, 0], [-np.sin(th), 0, np.cos(th)]], np.float32)
    tc = np.array([0.1, -0.2, 0.3], np.float32)
    pw = ((pc - tc) @ R.astype(np.float64)).astype(np.float32)
    q = rng.normal(size=(N, 4)).astype(np.float32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    s = (rng.uniform(0.01, 0.05, (N, 3)) * (0.2 if model == "ortho" else 1)).astype(np.float32)
    sh = (rng.normal(size=(N, 3 * k3)) * 0.3).astype(np.float32)
    return dict(pw=pw, q=q, s=s, sh=sh, R=R, t=tc, twc=(-R.T @ tc).astype(np.float32), intr=intr, W=W, H=H, N=N)


def _oracle_inputs(sc):
    """pc as camera_point rounds it in fp32 (each fmaf: an exact product and one rounding), so that rows near
    the axis, whose x / z the rounding of pc moves by ~1e-3, compare the same point; the covariance in fp64"""
    R = sc["R"].astype(np.float64)
    pw = sc["pw"].astype(np.float64)
    pc = np.empty_like(pw)
    for r in range(3):
        acc = np.float32(sc["t"][r]).astype(np.float64) + 0 * pw[:, 0]
        for c in (2, 1, 0):
            acc = (R[r, c] * pw[:, c] + acc).astype(np.float32).astype(np.float64)
        pc[:, r] = acc
    w, x, y, z = sc["q"].astype(np.float64).T
    Rq = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                   2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                   2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
    M = Rq * sc["s"].astype(np.float64)[:, None, :]
    S = M @ M.transpose(0, 2, 1)
    return pc, R, S[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]


@pytest.mark.parametrize("k3", [1, 4, 9, 16])
@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("model", oin.MODELS)
def test_host_backward_intrinsics_against_oracle(shim, model, aa, k3):
    """backward_one's 8 intrinsics terms per Gaussian (host build) against the oracle, each within 2e-5
    (pinhole) or 1e-4 (the lens models) of the sum of its terms' magnitudes; rows within 1e-4 of a cull or of the clamp bound (fp32 may put them on either
    side) are left out, culled rows must be exactly 0"""
    sc = _shim_scene(model, k3, 40 + k3 + 10 * MODEL_SEED[model])
    N = sc["N"]
    intr32 = np.asarray(sc["intr"], np.float32)
    lim = oin.limits(model, intr32, sc["W"], sc["H"])
    tan = np.array([lim[0] / 1.3, lim[1] / 1.3] if lim else [1.0, 1.0], np.float32)
    lim32 = (1.3 * float(tan[0]), 1.3 * float(tan[1])) if lim else None
    rng = np.random.default_rng(k3)
    gu = rng.normal(size=(N, 2)).astype(np.float32)
    gci = (rng.normal(size=(N, 3)) * 20).astype(np.float32)
    gcol = rng.normal(size=(N, 3)).astype(np.float32)
    gz = rng.normal(size=N).astype(np.float32)
    galpha = rng.normal(size=N).astype(np.float32)
    alphas = rng.uniform(0.2, 0.9, N).astype(np.float32)
    out = np.zeros((N, 23), np.float32)
    assert shim.intrinsics_backward_host(
        N, k3, MODEL_ID[model], int(aa), _p(sc["pw"]), _p(sc["q"]), _p(sc["s"]), _p(sc["sh"]), _p(sc["R"]),
        _p(sc["t"]), _p(sc["twc"]), *(C.c_float(v) for v in intr32[:4]), C.c_float(tan[0]), C.c_float(tan[1]),
        _p(intr32[4:].copy()), _p(gu), _p(gci), _p(gcol), _p(gz), _p(galpha), _p(alphas), _p(out)) == 0
    pc, R, c3 = _oracle_inputs(sc)
    keep = pc[:, 2] >= 0.2
    band = np.zeros(N, bool)
    if model == "fisheye":
        P1 = ocm.fisheye_terms(pc, intr32[4:])["P1"]
        keep &= P1 > 0
        band |= np.abs(P1) < 1e-4
    if model == "opencv":
        keep &= ocv.opencv_valid(pc, intr32[4:])[0]
        band |= ocv.opencv_band(pc, intr32[4:].astype(np.float64), *intr32[:4], sc["W"], sc["H"])
    if model == "pinhole":
        a, b = np.abs(pc[:, 0] / pc[:, 2]), np.abs(pc[:, 1] / pc[:, 2])
        band |= (np.abs(a - lim32[0]) < 1e-4 * lim32[0]) | (np.abs(b - lim32[1]) < 1e-4 * lim32[1])
    pe = np.where(keep[:, None], pc, [0.0, 0.0, 1.0])
    add = None
    if aa:
        c2 = oin._cov2d(oin.dproj(pe, model, intr32.astype(np.float64), lim32)[1], R, c3)[0]
        add = oaa.dcov2d_addend(c2, keep, alphas.astype(np.float64), galpha.astype(np.float64))
        band |= keep & oaa.scale(c2, keep)["clamped"]
    per, mag = oin.per_gaussian(pe, R, c3, model, intr32.astype(np.float64), lim32, gu, gci, add, keep,
                                magnitude=True)
    ok = ~band
    t = np.hypot(pc[:, 0], pc[:, 1]) / pc[:, 2]
    if model == "fisheye":
        # the series branch (t < 0.03) leaves out k3's and k4's terms of s and g, O(t^4) of k1's: there they
        # are held to k1's scale
        series = t < 0.03
        mag[series, 6:] = np.maximum(mag[series, 6:], mag[series, 4:5])
    got = out[:, 15:].astype(np.float64)
    err = np.abs(got - per)[ok]
    tol = 2e-5 if model == "pinhole" else 1e-4
    assert (err <= tol * mag[ok] + 1e-30).all(), (model, aa, k3, (err / (mag[ok] + 1e-30)).max())
    assert not got[~keep].any()
    if model in ("pinhole", "ortho"):
        assert not got[:, 4:].any()
    # what this scene was built to reach
    if model == "fisheye":
        assert ((t < 0.03) & keep & ok).sum() >= 40 and ((t > 0.03) & (t < 0.06) & keep & ok).sum() >= 40
    if model in ("pinhole", "opencv"):
        clamped = (np.abs(pc[:, 0] / pc[:, 2]) > lim32[0]) | (np.abs(pc[:, 1] / pc[:, 2]) > lim32[1])
        assert (clamped & keep & ok).sum() >= 10
    if model == "opencv":
        rho = t * t
        assert ((rho > 0.9 * ocv.opencv_rho_valid(*intr32[4:6])) & keep & ok).sum() >= 10


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("model", oin.MODELS)
def test_step_intrinsics_gradient_is_the_stage_derivative(model, aa):
    """oin.step on a 64-Gaussian RGB-D scene (64x48): its intrinsics gradient equals central differences of
    the per-Gaussian stages (u, conic, alpha_eff in fp64, clamp bound pinned) contracted with the rasterizer
    gradients step itself produced -- the loss the rasterizer backward linearises -- within 1e-6 of the sum of
    the contributions' magnitudes"""
    W, H = 64, 48
    k = {"fisheye": (0.05, -0.01, 0.0, 0.0), "opencv": (-0.08, 0.0, 0.0, 0.0)}.get(model)
    sc = camera_model_scene(64, W, H, model, radial_coeffs=(k if model == "fisheye" else (k[:2] if k else None)),
                            sh_dim=12, seed=3)
    cam = ost.camera(sc, W, H)
    rng = np.random.default_rng(1)
    dl = rng.normal(size=(3, H, W)).astype(np.float32)
    dld = rng.normal(size=(H, W)).astype(np.float32) * 0.1
    out = oin.step(sc, cam, rgbd=True, aa=aa, filt=None, dl=dl, dld=dld, model=model, k=k)
    st = out["st"]
    du, dc, da, _, _ = out["raster"]
    keep = np.asarray(st["keep"], bool)
    N = len(keep)
    kk = np.zeros(4) if k is None else np.asarray(k, np.float64)
    intr = np.array([float(np.float32(cam[n])) for n in ("fx", "fy", "cx", "cy")] + list(kk))
    lim = oin.limits(model, intr, W, H)
    pc = np.asarray(st["pcs"], np.float64)[keep]
    c3 = np.asarray(st["cov3ds"], np.float64)[keep]
    af = (np.asarray(out["drawn"]) / out["rho"])[keep]
    gu, gc, ga = np.asarray(du).reshape(N, 2)[keep], np.asarray(dc).reshape(N, 3)[keep], np.asarray(da).reshape(N)[keep]
    if aa:  # rows at the rho clamp have no rho derivative in the oracle
        sel = ~oaa.scale(st["c2"], keep)["clamped"][keep]
    else:
        sel = np.ones(len(pc), bool)

    def L(th):
        u, ci, rho = oin.forward(pc, cam["Rcw"], c3, model, th, lim)
        v = (gu * u).sum(1) + (gc * ci).sum(1) + (ga * af * rho if aa else 0.0)
        return v[sel].sum()

    want = out["iper"][keep][sel].sum(0)
    assert np.allclose(out["intr_grad"], out["iper"].sum(0)) and keep.sum() > 30
    for j in range(8 if model in ("fisheye", "opencv") else 4):
        h = 1e-6 * max(abs(intr[j]), 1.0)
        tp, tm = intr.copy(), intr.copy()
        tp[j] += h
        tm[j] -= h
        fd = (L(tp) - L(tm)) / (2 * h)
        assert abs(fd - want[j]) <= 1e-6 * out["iabsum"][j] + 1e-12, (model, aa, j, fd, want[j], out["iabsum"][j])


@pytest.fixture(scope="module")
def lib():
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    return _lib.load()


def test_workspace_queries(lib):
    q1 = lib.gsb_preprocess_backward_intrinsics_workspace_bytes
    for n in (0, 1, 128, 129, 20001):
        assert q1(n) == ((n + 127) // 128) * 96, n
    qb = lib.gsb_preprocess_backward_batch_intrinsics_workspace_bytes
    for Cn, N in ((1, 1), (3, 1000), (64, 1 << 24), (2, 0)):
        assert qb(Cn, N) == Cn * ((N + 127) // 128) * 96, (Cn, N)
    for Cn, N in ((0, 1000), (2, 1 << 30), (1, -1)):
        assert qb(Cn, N) == 0


def _err(lib):
    return lib.gsb_last_error().decode()


def test_argument_errors_before_any_launch(lib):
    store = (C.c_char * 8192)()
    buf = C.addressof(store) + (-C.addressof(store)) % 16
    f = buf + 64  # host addresses: nothing may be launched on them
    before = lib.gsb_profile_launches(-1)

    class CM(C.Structure):
        _fields_ = [("model", C.c_int32), ("k", C.c_float * 4)]

    def single(N=10, moments=True, dcam=True, dint=True, ws=None, ws_bytes=None, outs=None, cm=None, fx=100.0):
        need = lib.gsb_preprocess_backward_intrinsics_workspace_bytes(N)
        outs = [f] * 4 if outs is None else outs
        return lib.gsb_preprocess_backward_intrinsics(
            N, 16, *([f] * 7), fx, 100.0, 8.0, 8.0, 16.0, 16.0, None, None, None, *outs,
            f if moments else None, f, f, f, None, None, f if dcam else None, f if dint else None,
            buf if ws is None else ws, need if ws_bytes is None else ws_bytes,
            None if cm is None else C.byref(cm), None)

    cases = [
        (dict(moments=False), "null upstream gradient"),
        (dict(dcam=False), "null dloss_dcamera"),
        (dict(dint=False), "null dloss_dintrinsics"),
        (dict(ws=buf + 4), "misaligned"),
        (dict(ws_bytes=64), "too small"),
        (dict(N=1000, ws_bytes=7 * 96), "too small"),
        (dict(outs=[None, f, f, f]), "all set or all null"),
        (dict(cm=CM(0, (C.c_float * 4)(0.1, 0, 0, 0))), "fisheye and opencv"),
        (dict(cm=CM(1, (C.c_float * 4)(0, 0.1, 0, 0))), "fisheye and opencv"),
        (dict(cm=CM(4, (C.c_float * 4)(0.1, 0, 0, 0)), fx=-1.0), "fx and fy must be > 0"),
        (dict(cm=CM(7, (C.c_float * 4)(0, 0, 0, 0))), "unknown camera model"),
    ]
    for kw, msg in cases:
        rc = single(**kw)
        assert rc != 0 and msg in _err(lib), (kw, msg, _err(lib))
    rows = (C.c_float * 16)(200.0, 200.0, 8.0, 8.0, 0, 0, 0, 0, 210.0, 205.0, 8.0, 8.0, 0, 0, 0, 0)
    bad = (C.c_float * 16)(200.0, 200.0, 8.0, 8.0, 0, 0, 0, 0, 210.0, 205.0, 8.0, 8.0, 0.2, 0, 0, 0)

    def batch(Cn=2, N=10, intr=rows, model=0, dposes=True, dint=True, ws=None, ws_bytes=None):
        need = lib.gsb_preprocess_backward_batch_intrinsics_workspace_bytes(Cn, N)
        return lib.gsb_preprocess_backward_batch_intrinsics(
            Cn, N, 16, *([f] * 5), C.addressof(intr), model, 16.0, 16.0, f, f, None, None, *([f] * 6),
            f if dposes else None, f if dint else None, buf if ws is None else ws,
            need if ws_bytes is None else ws_bytes, None)

    bcases = [
        (dict(Cn=0), "C < 1"),
        (dict(Cn=65), "GSB_BATCH_MAX_CAMERAS"),
        (dict(dposes=False), "null dloss_dposes"),
        (dict(dint=False), "null dloss_dintrinsics"),
        (dict(ws=buf + 4), "misaligned"),
        (dict(ws_bytes=2 * 64), "too small"),
        (dict(intr=bad, model=0), "fisheye and opencv"),
        (dict(intr=bad, model=1), "fisheye and opencv"),
    ]
    for kw, msg in bcases:
        rc = batch(**kw)
        assert rc != 0 and msg in _err(lib), (kw, msg, _err(lib))
    assert lib.gsb_profile_launches(-1) == before


def test_python_argument_rules():
    from easygaussiansplatting_b200 import ops
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFusedBatchPose, GSFunctionFusedPose
    z = torch.zeros(0)
    with pytest.raises(ValueError, match="intrinsics_grad"):
        ops.preprocessB(*([z] * 4), torch.eye(3), torch.zeros(3), torch.zeros(3), 1.0, 1.0, 0.0, 0.0, 4, 4,
                        None, None, None, moments=torch.zeros(0, 9), cinv2ds=torch.zeros(0, 3), intrinsics_grad=True)
    with pytest.raises(ValueError, match="intrinsics_grad"):
        ops.preprocessB_batch(z, z, z, z, [Camera(4, 4, 1.0, 1.0, 2.0, 2.0, torch.eye(3), torch.zeros(3))], z, z,
                              intrinsics_grad=True)
    R, t = torch.eye(3), torch.zeros(3)
    cam = Camera(64, 48, 50.0, 50.0, 32.0, 24.0, R, t)
    N = 5
    g = [torch.zeros(N, 3), torch.zeros(N, 48), torch.zeros(N, 1), torch.zeros(N, 3), torch.zeros(N, 4),
         torch.zeros(N, 2)]
    for bad, msg in ((torch.zeros(7), "shape"), (torch.zeros(8, dtype=torch.int32), "float"),
                     (torch.tensor([50.0, 50, 32, 24, 0.1, 0, 0, 0]), "k must be 0"),
                     (torch.tensor([50.0, float("nan"), 32, 24, 0, 0, 0, 0]), "finite")):
        with pytest.raises(ValueError, match=msg):
            GSFunctionFusedPose.apply(*g, R, t, t, cam, None, None, bad)
    # the camera's other fields survive the replacement: the pose classes still refuse the exchange
    ex = Camera(64, 48, 50.0, 50.0, 32.0, 24.0, R, t)
    ex.grad_exchange = object()
    with pytest.raises(ValueError, match="single-view"):
        GSFunctionFusedPose.apply(*g, R, t, t, ex, None, None, torch.tensor([50.0, 50, 32, 24, 0, 0, 0, 0]))
    with pytest.raises(ValueError, match="shape"):
        GSFunctionFusedBatchPose.apply(*g[:5], torch.zeros(2, N, 2), torch.zeros(2, 3, 3), torch.zeros(2, 3),
                                       torch.zeros(2, 3), [cam, cam], None, torch.zeros(3, 8))


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not installed")
def test_new_kernels_in_the_cubin_without_stack_or_spills(lib):
    from easygaussiansplatting_b200 import _lib
    out = subprocess.run([CUOBJDUMP, "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    res = {k: v for k, v in re.findall(r"Function (\S+):\s*\n\s*(REG:\d+ STACK:\d+ SHARED:\d+ LOCAL:\d+)", out)}
    intr = [k for k in res if "k_preprocess_bwd_intrinsics" in k]
    red = [k for k in res if "k_intrinsics_reduce" in k]
    assert len(intr) == 64 and len(red) == 1  # K3 x DEPTH x AA x model; one reduction
    for k in intr + red:
        assert "STACK:0 " in res[k] and res[k].endswith("LOCAL:0"), (k, res[k])
        assert int(re.search(r"REG:(\d+)", res[k]).group(1)) <= 128, (k, res[k])
