"""CPU checks of the camera gradient (dL/dRcw, dL/dtcw, dL/dtwc): the fp64 pose oracle against
central differences of the whole RGB-D oracle chain, each Gaussian's contribution from the fused
backward (pg_fused_math.h through the host shim) against the oracle, the POSE kernels in the
sm_90a binary, and the workspace query."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import pose_oracle as opose
from oracle import rgbd_oracle as orgbd
from easygaussiansplatting_b200.scene import upstream_gradient

from test_fused_math_cpu import _p, _scene
from test_gpu_fused import scene as gpu_scene
from test_rgbd_cpu import _loss_rgbd, depth_shim  # noqa: F401  (depth_shim is a fixture)

HERE = os.path.dirname(os.path.abspath(__file__))
POSE_SO = os.path.join(HERE, "host_shim", "_build", "libfused_pose_host.so")


@pytest.fixture(scope="module")
def pose_shim():
    """tests/host_shim/fused_pose_host.cpp: backward_one with the camera gradient, host build"""
    src = os.path.join(HERE, "host_shim", "fused_pose_host.cpp")
    hdr = os.path.join(HERE, "..", "easygaussiansplatting_b200", "csrc", "pg_fused_math.h")
    os.makedirs(os.path.dirname(POSE_SO), exist_ok=True)
    if not os.path.exists(POSE_SO) or os.path.getmtime(POSE_SO) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", POSE_SO, src],
                       check=True)
    return C.CDLL(POSE_SO)


def _cone_scene(N, W, H, seed):
    """test_gpu_fused.scene's rotated camera (odd seed), keeping only the Gaussians well inside the
    1.3 tan_fov cone and in front of the near plane: there the oracle's chain is smooth in the pose"""
    sc = gpu_scene(N, W, H, 48, seed)
    pc = sc["pws"].astype(np.float64) @ sc["Rcw"].astype(np.float64).T + sc["tcw"]
    tx, ty = W / (2 * sc["fx"]), H / (2 * sc["fy"])
    z = pc[:, 2]
    keep = (z > 0.5) & (np.abs(pc[:, 0]) < 1.1 * tx * z) & (np.abs(pc[:, 1]) < 1.1 * ty * z)
    out = {}
    for k, v in sc.items():
        if isinstance(v, np.ndarray) and v.ndim >= 1 and v.shape[0] == N and k not in ("Rcw", "tcw", "twc"):
            v = v[keep]
        out[k] = np.array(v, dtype=np.float64) if isinstance(v, np.ndarray) else v
    return out


def _oracle_camera_grad(sc, W, H, G):
    st = opose.stages(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                      sc["fy"], sc["cx"], sc["cy"], W, H)
    fwd = orgbd.splat_rgbd(H, W, st["us"], st["ci"], sc["alphas"], st["depths"].copy(), st["col"],
                           st["areas"].copy())
    du, dc, _, dcol, dz = orgbd.splat_backward_rgbd(H, W, st["us"], st["ci"], sc["alphas"], st["col"], fwd["z"], fwd,
                                                    G[0], G[1], G[2])
    return opose.camera_grad(st, sc["pws"], sc["Rcw"], sc["fx"], sc["fy"], W, H, du, dc, dcol, dz)


def _stage_loss(sc, W, H, up):
    """the per-Gaussian stages' outputs contracted with fixed upstream gradients: the loss the
    rasterizer backward linearises"""
    st = opose.stages(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                      sc["fy"], sc["cx"], sc["cy"], W, H)
    du, dc, dcol, dz = up
    z = np.where(st["keep"], st["pcs"][:, 2].astype(np.float64), 0.0)
    return float((du.reshape(-1, 2) * st["us"]).sum() + (dc.reshape(-1, 3) * st["ci"]).sum() +
                 (dcol.reshape(-1, 3) * st["col"]).sum() + (dz * z).sum())


def _central(f, x, j, rel):
    x0 = float(x[j])
    h = rel * max(abs(x0), 0.05)
    # the stages read fp32: both points are fp32 values and the difference is taken between them
    xp, xm = float(np.float32(x0 + h)), float(np.float32(x0 - h))
    x[j] = xp
    lp = f()
    x[j] = xm
    lm = f()
    x[j] = x0
    return (lp - lm) / (xp - xm)


def _fd_checks(seed, W, H):
    sc = _cone_scene(200, W, H, seed)
    assert len(sc["pws"]) > 100 and not np.allclose(sc["Rcw"], np.eye(3))
    rng = np.random.default_rng(seed + 7)
    G = (upstream_gradient(W, H, seed).astype(np.float64) * (3.0 * W * H),
         rng.normal(size=(H, W)) * 0.3, rng.normal(size=(H, W)))
    loss, (us, ci, col, fwd, _) = _loss_rgbd(sc, W, H, G)
    du, dc, _, dcol, dz = orgbd.splat_backward_rgbd(H, W, us, ci, sc["alphas"], col, fwd["z"], fwd, G[0], G[1], G[2])
    up = (du, dc, dcol, dz)
    an = _oracle_camera_grad(sc, W, H, G)["grad"]
    good, full_fd = [], []
    for e in range(15):
        name, j = ("Rcw", e) if e < 9 else (("tcw", e - 9) if e < 12 else ("twc", e - 12))
        x = sc[name].reshape(-1)
        ok = False
        for rel in (2e-3, 5e-4, 1.5e-4):  # three step sizes (test_oracle_fd.py)
            fd = _central(lambda: _stage_loss(sc, W, H, up), x, j, rel)
            if abs(fd - an[e]) <= 1e-2 * max(abs(fd), abs(an[e])) + 1e-9 * abs(loss):
                ok = True
                break
        good.append(ok)
        full_fd.append(_central(lambda: _loss_rgbd(sc, W, H, G)[0], x, j, 1e-2))
    assert np.abs(an[12:]).max() > 0 and np.abs(an[:9]).max() > 0
    return good, np.array(full_fd), an


def test_camera_gradient_vs_central_differences():
    """L = <G1, image> + <G2, D> + <G3, A> through the RGB-D oracle chain, on two seeds with a
    general pose; Rcw, tcw and twc are each perturbed on their own.
    - The pose oracle's 15 entries against central differences of the per-Gaussian stages
      (project ... inverse_cov2d) contracted with the rasterizer backward's dL/du, dL/dconic,
      dL/dcolour, dL/dz of L: the camera's whole chain below the rasterizer, whose own backward
      test_rgbd_cpu differentiates.  At least 90 % of the 30 checks agree.
    - Central differences of L itself: moving the camera moves every Gaussian at once, so many
      pixels cross the 1/255 opacity threshold within one step and each crossing is a jump; the
      whole 15-vector still has to agree to 25 % in norm (a wrong sign or term is far off)."""
    g1, f1, a1 = _fd_checks(11, 64, 48)
    g2, f2, a2 = _fd_checks(13, 64, 48)
    good = g1 + g2
    assert sum(good) >= 27, "%d of 30 camera entries agree (%s)" % (sum(good), good)
    for fd, an in ((f1, a1), (f2, a2)):
        assert np.linalg.norm(fd - an) <= 0.25 * np.linalg.norm(an), (fd, an)


@pytest.mark.parametrize("k3", [1, 4, 9, 16])
def test_fused_backward_camera_terms_match_oracle(pose_shim, depth_shim, k3):  # noqa: F811
    W, H, N = 320, 240, 3000
    sc = _scene(N, k3, seed=50 + k3)
    st = opose.stages(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                      sc["fy"], sc["cx"], sc["cy"], W, H)
    keep = st["keep"]
    assert (~keep).any() and keep.any()
    # rows with the fov clamp active (_scene widens some): J uses the clamped x, y there
    pc = st["pcs"].astype(np.float64)
    clamped = keep & (np.abs(pc[:, 0]) > 1.3 * W / (2 * sc["fx"]) * pc[:, 2])
    assert clamped.any()
    rng = np.random.default_rng(k3 + 200)
    gu = rng.normal(size=(N, 2)).astype(np.float32)
    gci = (rng.normal(size=(N, 3)) * 10).astype(np.float32)
    gcol = rng.normal(size=(N, 3)).astype(np.float32)
    gz = rng.normal(size=N).astype(np.float32)
    ref = opose.camera_grad(st, sc["pws"], sc["Rcw"], sc["fx"], sc["fy"], W, H, gu, gci, gcol, gz)["per"]
    out = {k: np.empty(s, np.float32) for k, s in (("pws", (N, 3)), ("shs", (N, 3 * k3)), ("scales", (N, 3)),
                                                   ("rots", (N, 4)), ("cam", (N, 15)))}
    args = [_p(sc["pws"]), _p(sc["rots"]), _p(sc["scales"]), _p(sc["shs"]), _p(sc["Rcw"]), _p(sc["tcw"]),
            _p(sc["twc"]), C.c_float(sc["fx"]), C.c_float(sc["fy"]), C.c_float(sc["cx"]), C.c_float(sc["cy"]),
            C.c_float(W), C.c_float(H), _p(gu), _p(gci), _p(gcol), _p(gz)]
    assert pose_shim.fused_backward_pose_host(N, k3, *args, *[_p(out[k]) for k in ("pws", "shs", "scales", "rots",
                                                                                  "cam")]) == 0
    for c in range(15):
        s = np.abs(ref[:, c]).max()
        if s == 0:  # dL/dtwc at SH degree 0
            assert c >= 12 and k3 == 1 and not out["cam"][:, c].any()
            continue
        e = np.abs(out["cam"][:, c].astype(np.float64) - ref[:, c]).max() / s
        assert e <= 2e-5, (c, e)
    # culled rows: the colour branch only
    assert not out["cam"][~keep, :12].any()
    if k3 > 1:
        assert np.abs(out["cam"][~keep, 12:]).max() > 0
    # the per-Gaussian outputs are those of the non-POSE instantiation, bit for bit
    base = {k: np.empty_like(out[k]) for k in ("pws", "shs", "scales", "rots")}
    assert depth_shim.fused_backward_depth_host(N, k3, *args, *[_p(base[k]) for k in ("pws", "shs", "scales",
                                                                                     "rots")]) == 0
    for k in base:
        assert np.array_equal(out[k].view(np.uint32), base[k].view(np.uint32)), k


def test_pose_kernels_are_sm90a_without_spills():
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    r = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True)
    assert r.returncode == 0
    found = {}
    for name, usage in re.findall(r"Function (_ZN3gsb16k_preprocess_bwd\S+):\s*\n\s*(REG:.*)", r.stdout):
        t = re.search(r"ILi(\d+)ELb(\d)ELb(\d)ELb(\d)ELb(\d)E", name).groups()
        if t[4] == "1":
            found[t[:4]] = usage
    # POSE is built for every K3 with MOM x DEPTH, never with PUSH
    want = {(k, "0", m, d) for k in ("1", "4", "9", "16") for m in "01" for d in "01"}
    assert set(found) == want
    for t, usage in found.items():
        assert "STACK:0 " in usage and "LOCAL:0 " in usage, (t, usage)
    r = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True)
    assert "_ZN3gsb13k_pose_reduce" in r.stdout
    assert re.search(r"arch = sm_90a", r.stdout)


def test_pose_workspace_query_without_gpu():
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    lib = _lib.load()
    for n, want in ((0, 0), (1, 64), (128, 64), (129, 128), (20001, 157 * 64), (1000000, 7813 * 64)):
        assert lib.gsb_preprocess_backward_pose_workspace_bytes(n) == want, n
