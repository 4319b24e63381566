"""The 2D Gaussian Splatting math of the surfel kernels (surfel_math.h), run on the host through
tests/host_shim/surfel_host.cpp, against the fp64 oracle (oracle/surfel_oracle.py): the per-surfel
forward (us, depths, areas, colours, records), the per-surfel backward from gradient rows, the
per-pixel evaluation and its gradient (central differences of the oracle's evaluation, dL/du folded
into dL/dM), and the cull box (no pixel outside it reaches alpha' >= 0.002)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import surfel_oracle as so

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "host_shim", "_build", "libsurfel_host.so")
FX, FY, CX, CY = 300.0, 280.0, 161.3, 119.6


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def shim():
    src = os.path.join(HERE, "host_shim", "surfel_host.cpp")
    hdrs = [os.path.join(HERE, "..", "easygaussiansplatting_b200", "csrc", h) for h in ("surfel_math.h", "pg_fused_math.h")]
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(f) for f in [src] + hdrs):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", SO, src], check=True)
    lib = C.CDLL(SO)
    f = C.c_float
    lib.surfel_forward.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 8 + [f] * 4 + [C.c_void_p] * 5
    lib.surfel_backward.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 7 + [f] * 4 + [C.c_void_p] * 5
    lib.surfel_pixel.argtypes = [C.c_void_p, C.c_void_p, f, f, f, f, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.surfel_extents.argtypes = [C.c_void_p, C.c_void_p, f, f, C.c_void_p, C.c_void_p]
    return lib


def f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def scene(N, k, seed):
    rng = np.random.default_rng(seed)
    z = rng.uniform(0.5, 8.0, N)
    pws = np.stack([rng.uniform(-1, 1, N) * z * 0.5, rng.uniform(-1, 1, N) * z * 0.4, z], 1)
    rots = rng.normal(size=(N, 4))
    scales = np.stack([rng.uniform(0.01, 0.3, N), rng.uniform(0.01, 0.3, N), rng.uniform(0, 0.1, N)], 1)
    th = 0.3
    Rcw = np.array([[np.cos(th), 0, np.sin(th)], [0, 1, 0], [-np.sin(th), 0, np.cos(th)]])
    twc = np.array([0.1, -0.2, 0.05])
    tcw = -Rcw @ twc
    pws[0] = Rcw.T @ (np.array([0.01, 0.01, 0.15]) - tcw)  # culled: camera z < 0.2
    # edge-on: the world normal R e2 lies along the camera's x axis, the surfel on the optical axis
    pws[1] = Rcw.T @ (np.array([0.0, 0.0, 2.0]) - tcw)
    Rw = Rcw.T @ np.array([[0, 0, 1], [0, 1, 0], [-1, 0, 0.0]])  # columns: R e0, R e1, R e2 = Rcw^T e_x
    w = np.sqrt(max(1e-12, 1 + np.trace(Rw))) / 2
    rots[1] = [w, (Rw[2, 1] - Rw[1, 2]) / (4 * w), (Rw[0, 2] - Rw[2, 0]) / (4 * w), (Rw[1, 0] - Rw[0, 1]) / (4 * w)]
    return dict(pws=f32(pws), rots=f32(rots), scales=f32(scales), shs=f32(rng.normal(scale=0.3, size=(N, 3 * k))),
                alphas=f32(rng.uniform(0.001, 0.999, N)), Rcw=f32(Rcw), tcw=f32(tcw), twc=f32(twc))


def shim_forward(lib, sc, k):
    N = len(sc["pws"])
    us, depths, cols = np.zeros((N, 2), np.float32), np.zeros(N, np.float32), np.zeros((N, 3), np.float32)
    areas, recs = np.zeros((N, 2), np.int32), np.zeros((N, 20), np.float32)
    assert lib.surfel_forward(N, k, *[_p(sc[n]) for n in ("pws", "rots", "scales", "shs", "alphas", "Rcw", "tcw", "twc")],
                              FX, FY, CX, CY, _p(us), _p(depths), _p(areas), _p(cols), _p(recs)) == 0
    return us, depths, areas, cols, recs


def oracle_pre(sc):
    return so.preprocess(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], FX, FY, CX, CY)


@pytest.mark.parametrize("k", [1, 4, 9, 16])
def test_forward_matches_oracle_stages(shim, k):
    sc = scene(400, k, seed=k)
    us, depths, areas, cols, recs = shim_forward(shim, sc, k)
    pre = oracle_pre(sc)
    keep = pre["keep"]
    assert not keep[0] and keep.sum() > 300
    assert ((depths == -1) == ~keep).all() and (areas[~keep] == 0).all() and (recs[~keep, 9] == 0).all()
    np.testing.assert_allclose(depths[keep], pre["depths"][keep], rtol=1e-6)
    np.testing.assert_allclose(us[keep], pre["u"][keep], rtol=1e-5, atol=1e-3)
    np.testing.assert_allclose(cols, pre["colors"], atol=2e-5)
    M = pre["M"].reshape(-1, 9)
    scale = np.abs(M).max(axis=1, keepdims=True)
    assert (np.abs(recs[keep, :9] - M[keep]) <= 2e-6 * scale[keep]).all()
    np.testing.assert_allclose(recs[keep, 9], sc["alphas"][keep])
    np.testing.assert_allclose(recs[keep, 10:12], us[keep])
    np.testing.assert_allclose(recs[keep, 14:17], cols[keep], atol=0)
    np.testing.assert_allclose(recs[keep, 17:20], pre["n"][keep], atol=2e-6)
    # integer footprints: equal to the oracle's except where its ceil sits within fp32 rounding of an integer
    ext, _ = so.footprint(pre["M"], pre["u"], so.CUTOFF2)
    near = np.abs(ext - np.round(ext)) < 1e-4 * np.maximum(1, ext)
    assert ((areas[keep] == pre["areas"][keep]) | near[keep]).all()


@pytest.mark.parametrize("k", [1, 4, 9, 16])
def test_backward_matches_oracle(shim, k):
    sc = scene(300, k, seed=10 + k)
    N = len(sc["pws"])
    rng = np.random.default_rng(k)
    rows = f32(rng.normal(size=(N, 18)))
    gpw, gsh = np.zeros((N, 3), np.float32), np.zeros((N, 3 * k), np.float32)
    gs, gq = np.zeros((N, 3), np.float32), np.zeros((N, 4), np.float32)
    assert shim.surfel_backward(N, k, *[_p(sc[n]) for n in ("pws", "rots", "scales", "shs", "Rcw", "tcw", "twc")],
                                FX, FY, CX, CY, _p(rows), _p(gpw), _p(gsh), _p(gs), _p(gq)) == 0
    ref = so.preprocess_backward(oracle_pre(sc), rows.astype(np.float64))
    for name, got in (("pws", gpw), ("shs", gsh), ("scales", gs), ("rots", gq)):
        want = ref[name]
        err = np.abs(got - want).max() / np.abs(want).max()
        assert err < 2e-5, (name, err)
    assert (gs[:, 2] == 0).all()


def _oracle_L(M, x, y, dG, dz, delta=(0.0, 0.0)):
    u = np.array([M[0, 2] / M[2, 2], M[1, 2] / M[2, 2]])
    e = so._eval(M, u, np.array([x - delta[0]]), np.array([y - delta[1]]))
    return dG * e["G"][0] + dz * e["z"][0], e


def test_pixel_eval_and_gradient(shim):
    rng = np.random.default_rng(5)
    sc = scene(200, 1, seed=5)
    pre = oracle_pre(sc)
    _, _, _, _, recs = shim_forward(shim, sc, 1)
    seen = {True: 0, False: 0}
    for i in np.flatnonzero(pre["keep"]):
        if i == 1:
            continue  # edge-on: c2 ~ 0, G3 swings across G2 under any perturbation of m3
        M = recs[i, :9].astype(np.float64).reshape(3, 3)
        u = np.array([M[0, 2] / M[2, 2], M[1, 2] / M[2, 2]])
        ext, ok = so.footprint(M[None], u[None], 9.0)
        if not ok[0]:
            continue
        x, y = float(np.round(u[0] + rng.uniform(-1.2, 1.2) * ext[0, 0])), float(np.round(u[1] + rng.uniform(-1.2, 1.2) * ext[0, 1]))
        dG, dz = rng.normal(), rng.normal()
        M32 = f32(M.ravel())
        u32 = f32(u)
        out, gM, gd = np.zeros(4, np.float32), np.zeros(9, np.float32), np.zeros(2, np.float32)
        shim.surfel_pixel(_p(M32), _p(u32), x, y, dG, dz, _p(out), _p(gM), _p(gd))
        L0, e = _oracle_L(M, x, y, dG, dz)
        if abs(e["G3"][0] - e["G2"][0]) < 1e-3 * max(1.0, e["G2"][0]) or not np.isfinite(e["G3"][0]):
            continue  # at the switch of the two terms (and edge-on, c2 = 0) it is not differentiable
        assert bool(out[2]) == bool(e["b3"][0])
        np.testing.assert_allclose(out[0], e["G"][0], rtol=1e-3, atol=1e-4)
        np.testing.assert_allclose(out[1], e["z"][0], rtol=1e-4)
        h = 1e-9 * np.abs(M).max()
        fd = np.zeros(9)
        for j in range(9):
            Mp, Mm = M.copy(), M.copy()
            Mp.flat[j] += h
            Mm.flat[j] -= h
            fd[j] = (_oracle_L(Mp, x, y, dG, dz)[0] - _oracle_L(Mm, x, y, dG, dz)[0]) / (2 * h)
        fdd = np.array([(_oracle_L(M, x, y, dG, dz, (s * 1e-6, 0))[0] - _oracle_L(M, x, y, dG, dz, (-s * 1e-6, 0))[0])
                        for s in (1,)] + [(_oracle_L(M, x, y, dG, dz, (0, 1e-6))[0] -
                                           _oracle_L(M, x, y, dG, dz, (0, -1e-6))[0])]) / 2e-6
        sg = np.abs(fd).max()
        assert np.abs(gM - fd).max() <= 2e-4 * sg + 1e-6, (i, gM, fd)
        assert np.abs(gd - fdd).max() <= 2e-4 * max(np.abs(fdd).max(), 1e-6), (i, gd, fdd)
        seen[bool(out[2])] += 1
    assert seen[True] > 50 and seen[False] > 5


def test_cull_box_holds_every_reachable_pixel(shim):
    """outside the record's cull box no pixel reaches min(G3, G2) <= 2 ln(alpha / 0.002)"""
    rng = np.random.default_rng(9)
    sc = scene(300, 1, seed=9)
    pre = oracle_pre(sc)
    _, _, _, _, recs = shim_forward(shim, sc, 1)
    checked = 0
    for i in np.flatnonzero(pre["keep"]):
        M32, u32 = f32(recs[i, :9]), f32(recs[i, 10:12])
        cull, ext = np.zeros(2, np.float32), np.zeros(2, np.float32)
        shim.surfel_extents(_p(M32), _p(u32), float(sc["alphas"][i]), 9.0, _p(cull), _p(ext))
        np.testing.assert_array_equal(cull, recs[i, 12:14])
        if not np.isfinite(cull).all():
            continue
        t = 2 * np.log(sc["alphas"][i] / 0.002)
        span = np.maximum(cull, 1.0) * 2.5
        X = np.floor(u32[0] + rng.uniform(-span[0], span[0], 4000))
        Y = np.floor(u32[1] + rng.uniform(-span[1], span[1], 4000))
        e = so._eval(M32.astype(np.float64).reshape(3, 3), u32.astype(np.float64), X, Y)
        inside = (np.abs(X - u32[0]) <= cull[0]) & (np.abs(Y - u32[1]) <= cull[1])
        assert not ((e["G"] <= t) & ~inside).any(), i
        checked += 1
    assert checked > 100
