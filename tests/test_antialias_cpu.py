"""CPU checks of antialiasing (the 2D-filter opacity compensation alpha_eff = rho alpha): the fp64
oracle (oracle/aa_oracle.py) against central differences, the host build of the fused forward and
backward's AA forms (pg_fused_math.h through tests/host_shim/fused_aa_host.cpp) against the oracle
at every SH degree and on edge rows, the kernels' forms in the sm_90a binary, and the property the
feature exists for: coverage that stays put when a scene is rendered smaller."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import aa_oracle as oaa
from oracle import oracle as orc
from oracle import pose_oracle as opose

from test_fused_math_cpu import _p, _scene, shim  # noqa: F401  (shim is a fixture)

HERE = os.path.dirname(os.path.abspath(__file__))
AA_SO = os.path.join(HERE, "host_shim", "_build", "libfused_aa_host.so")
W, H = 320, 240


@pytest.fixture(scope="module")
def aa_shim():
    src = os.path.join(HERE, "host_shim", "fused_aa_host.cpp")
    hdr = os.path.join(HERE, "..", "easygaussiansplatting_b200", "csrc", "pg_fused_math.h")
    os.makedirs(os.path.dirname(AA_SO), exist_ok=True)
    if not os.path.exists(AA_SO) or os.path.getmtime(AA_SO) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", AA_SO, src],
                       check=True)
    return C.CDLL(AA_SO)


def edge_scene(k3, seed, n=3000):
    """_scene (culled rows, fov-clamped rows, a general camera) with the AA edge rows at its head:
    0-3 zero scale (r = 0: the clamp holds), 4-7 needles (large kappa), 8-11 huge (rho -> 1),
    12-15 culled (rho = 1).  -> (scene, dict of row index arrays)"""
    return aa_edge_rows(_scene(n, k3, seed=seed))


def aa_edge_rows(sc):
    """edge_scene's head rows written into any scene (in place) -> (scene, dict of row index arrays)"""
    pc_mid = sc["pws"][sc["pws"][:, 2] > 0][:16]
    sc["pws"][:16] = pc_mid
    sc["scales"][0:4] = 0.0
    sc["scales"][4:8] = np.array([0.4, 2e-4, 2e-4], np.float32)
    sc["scales"][8:12] = 6.0
    sc["pws"][12:16] = np.array([0.0, 0.0, -5.0], np.float32)  # far behind the camera
    rows = dict(zero=np.arange(0, 4), needle=np.arange(4, 8), huge=np.arange(8, 12), culled=np.arange(12, 16))
    return sc, rows


def _cam_args(sc):
    return [_p(sc["pws"]), _p(sc["rots"]), _p(sc["scales"]), _p(sc["shs"]), _p(sc["Rcw"]), _p(sc["tcw"]),
            _p(sc["twc"]), C.c_float(sc["fx"]), C.c_float(sc["fy"]), C.c_float(sc["cx"]), C.c_float(sc["cy"]),
            C.c_float(W), C.c_float(H)]


def host_forward(lib, sc, k3, aa):
    N = len(sc["pws"])
    o = dict(us=np.empty((N, 2), np.float32), ci=np.empty((N, 3), np.float32), col=np.empty((N, 3), np.float32),
             d=np.empty(N, np.float32), ar=np.empty((N, 2), np.int32))
    outs = [_p(o[k]) for k in ("us", "ci", "col", "d", "ar")]
    if aa:
        o["rho"] = np.empty(N, np.float32)
        assert lib.fused_forward_aa_host(N, k3, *_cam_args(sc), *outs, _p(o["rho"])) == 0
    else:
        assert lib.fused_forward_host(N, k3, *_cam_args(sc), *outs) == 0
    return o


def host_backward(lib, sc, k3, up, pose):
    N = len(sc["pws"])
    o = {k: np.empty(s, np.float32) for k, s in (("pws", (N, 3)), ("shs", (N, 3 * k3)), ("scales", (N, 3)),
                                                 ("rots", (N, 4)), ("alphas", (N,)), ("cam", (N, 15)))}
    gu, gci, gcol, gz, gal = up
    assert lib.fused_backward_aa_host(N, k3, *_cam_args(sc), _p(gu), _p(gci), _p(gcol), _p(gz), _p(gal),
                                      _p(sc["alphas"]), *[_p(o[k]) for k in ("pws", "shs", "scales", "rots", "alphas")],
                                      _p(o["cam"]) if pose else None) == 0
    return o


def oracle_backward(sc, k3, up):
    """the oracle chain of the non-AA upstream gradients plus the AA addend -> (dict, stages, scale)"""
    gu, gci, gcol, gz, gal = (np.asarray(a, np.float64) for a in up)
    N = len(sc["pws"])
    st = oaa.stages(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                    sc["fy"], sc["cx"], sc["cy"], W, H)
    keep = st["keep"]
    s = oaa.scale(st["c2"], keep)
    gz_keep = np.where(keep, gz, 0.0)
    base = orc.chain_backward(sc["Rcw"], gu.reshape(N, 1, 2), gci.reshape(N, 1, 3), gal.reshape(N, 1, 1),
                              gcol.reshape(N, 1, 3), *st["J"])
    # the depth term: dL/dpc[2] = gz on kept rows, rotated by Rcw
    base["pws"] = base["pws"] + gz_keep[:, None] * np.asarray(sc["Rcw"], np.float64)[2][None, :]
    gc2 = oaa.dcov2d_addend(st["c2"], keep, sc["alphas"], gal)
    add = oaa.chain(st, sc["Rcw"], gc2)
    ref = {k: base[k] + add[k] for k in ("pws", "scales", "rots")}
    ref["shs"] = base["shs"]
    ref["alphas"] = s["rho"] * gal
    cam = opose.camera_grad(st, sc["pws"], sc["Rcw"], sc["fx"], sc["fy"], W, H, gu, gci, gcol, gz)["per"]
    ref["cam"] = cam + oaa.camera(st, sc["pws"], sc["Rcw"], sc["fx"], sc["fy"], W, H, gc2)
    return ref, st, s, gc2


def upstream(sc, k3, seed, rows=None):
    N = len(sc["pws"])
    rng = np.random.default_rng(seed)
    gu = rng.normal(size=(N, 2)).astype(np.float32)
    gci = (rng.normal(size=(N, 3)) * 10).astype(np.float32)
    gcol = rng.normal(size=(N, 3)).astype(np.float32)
    gz = rng.normal(size=N).astype(np.float32)
    gal = (rng.normal(size=N) * 3).astype(np.float32)
    sc["alphas"] = rng.uniform(0.05, 1.0, N).astype(np.float32)
    if rows is not None:  # rows whose only upstream gradient is dL/dalpha_eff
        gu[rows] = 0; gci[rows] = 0; gcol[rows] = 0; gz[rows] = 0
    return gu, gci, gcol, gz, gal


rel_tol = oaa.rel_tol  # (the tolerance of an fp32 rho, shared with oracle/step_oracle.py)


# ---------------------------------------------------------------- the oracle itself
def test_oracle_rho_gradient_vs_central_differences():
    """dcov2d_addend (alpha = galpha = 1 -> drho/d(a', b, c')) against central differences of rho on
    well-conditioned random pre-blur covariances, on both sides of rho's range; the clamp's rows get 0"""
    rng = np.random.default_rng(3)
    n = 400
    L = rng.normal(size=(n, 2, 2)) * rng.choice([0.05, 0.3, 1.0, 4.0], size=(n, 1, 1))
    S = L @ L.transpose(0, 2, 1) + 1e-3 * np.eye(2)
    c2 = np.stack([S[:, 0, 0] + 0.3, S[:, 0, 1], S[:, 1, 1] + 0.3], axis=1)
    keep = np.ones(n, bool)
    s = oaa.scale(c2, keep)
    sel = (s["r"] > 1e-3) & (s["kappa"] < 100)  # away from the clamp, well conditioned
    c2, keep, n = c2[sel], keep[sel], int(sel.sum())
    s = oaa.scale(c2, keep)
    assert n > 200 and s["rho"].min() < 0.1 and s["rho"].max() > 0.9
    an = oaa.dcov2d_addend(c2, keep, np.ones(n), np.ones(n))
    for j in range(3):
        h = 1e-6 * np.maximum(np.abs(c2[:, j]), 1e-2)
        cp, cm = c2.copy(), c2.copy()
        cp[:, j] += h; cm[:, j] -= h
        fd = (oaa.scale(cp, keep)["rho"] - oaa.scale(cm, keep)["rho"]) / (2 * h)
        assert np.allclose(an[:, j], fd, rtol=1e-5, atol=1e-8 * np.abs(fd).max()), j
    # the clamp: r <= 2.5e-5 -> rho = 0.005 and no gradient; culled rows: rho = 1, no gradient
    tiny = np.array([[0.3 + 1e-6, 0.0, 0.3 + 1e-6], [0.3, 0.0, 0.3], [0.0, 0.0, 0.0]])
    s = oaa.scale(tiny, np.array([True, True, False]))
    assert np.allclose(s["rho"], [0.005, 0.005, 1.0]) and list(s["clamped"]) == [True, True, False]
    assert not oaa.dcov2d_addend(tiny, np.array([True, True, False]), np.ones(3), np.ones(3)).any()


def test_oracle_chain_vs_central_differences():
    """L = sum_i alpha_i galpha_i rho_i(pw, s, q) through the oracle's stages: the chained addend
    against central differences in the parameters of Gaussians away from the clamp and the fov edge"""
    k3 = 4
    sc = _scene(300, k3, seed=21)
    N = len(sc["pws"])
    rng = np.random.default_rng(22)
    sc["scales"] = (sc["scales"] * rng.uniform(0.05, 1.0, (N, 1))).astype(np.float32)  # many sub-pixel rows
    alphas = rng.uniform(0.1, 1.0, N)
    gal = rng.normal(size=N)

    def loss():
        st = oaa.stages(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                        sc["fy"], sc["cx"], sc["cy"], W, H)
        return float((alphas * gal * oaa.scale(st["c2"], st["keep"])["rho"]).sum()), st

    _, st = loss()
    s = oaa.scale(st["c2"], st["keep"])
    pc = st["pcs"].astype(np.float64)
    inside = st["keep"] & (np.abs(pc[:, 0]) < 1.2 * W / (2 * sc["fx"]) * pc[:, 2]) & \
        (np.abs(pc[:, 1]) < 1.2 * H / (2 * sc["fy"]) * pc[:, 2]) & (s["r"] > 1e-3) & (s["kappa"] < 1e3)
    assert inside.sum() > 50 and s["rho"][inside].min() < 0.5
    an = oaa.chain(st, sc["Rcw"], oaa.dcov2d_addend(st["c2"], st["keep"], alphas, gal))
    good = total = 0
    for i in np.flatnonzero(inside)[:12]:
        for name, m in (("pws", 3), ("scales", 3), ("rots", 4)):
            for j in range(m):
                x = sc[name][i]
                x0 = float(x[j])
                ok = False
                for rel in (1e-2, 3e-3, 1e-3):
                    h = rel * max(abs(x0), 0.05)
                    xp, xm = float(np.float32(x0 + h)), float(np.float32(x0 - h))
                    x[j] = xp; lp = loss()[0]
                    x[j] = xm; lm = loss()[0]
                    x[j] = x0
                    fd = (lp - lm) / (xp - xm)
                    a = an[name][i, j]
                    if abs(fd - a) <= 2e-2 * max(abs(fd), abs(a)) + 1e-7:
                        ok = True
                        break
                good += ok
                total += 1
    assert good >= 0.9 * total, "%d of %d chained entries agree" % (good, total)


# ---------------------------------------------------------------- host build vs oracle
@pytest.mark.parametrize("k3", [1, 4, 9, 16])
def test_host_forward_aa_matches_oracle(aa_shim, shim, k3):  # noqa: F811
    sc, rows = edge_scene(k3, seed=60 + k3)
    got = host_forward(aa_shim, sc, k3, aa=True)
    base = host_forward(shim, sc, k3, aa=False)
    for k in ("us", "ci", "col", "d", "ar"):  # every other output: the non-AA bits
        assert np.array_equal(got[k].view(np.uint32), base[k].view(np.uint32)), k
    st = oaa.stages(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                    sc["fy"], sc["cx"], sc["cy"], W, H)
    s = oaa.scale(st["c2"], st["keep"])
    tol = s["rho"] * rel_tol(s)
    err = np.abs(got["rho"].astype(np.float64) - s["rho"])
    ok = (err <= tol) | s["near"]
    assert ok.all(), (np.flatnonzero(~ok)[:5], err[~ok][:5], tol[~ok][:5])
    assert np.all(got["rho"][rows["zero"]] == np.float32(np.sqrt(np.float32(2.5e-5))))
    assert s["kappa"][rows["needle"]].min() > 1e3
    assert got["rho"][rows["huge"]].min() > 0.99
    assert np.all(got["rho"][rows["culled"]] == 1.0) and np.all(got["rho"][~st["keep"]] == 1.0)
    assert (got["rho"] <= 1.0).all() and got["rho"].min() < 0.1


@pytest.mark.parametrize("k3", [1, 4, 9, 16])
@pytest.mark.parametrize("pose", [False, True])
def test_host_backward_aa_matches_oracle(aa_shim, k3, pose):
    sc, rows = edge_scene(k3, seed=70 + k3)
    only = np.arange(16, 64)  # rows whose only upstream gradient is dL/dalpha_eff
    up = upstream(sc, k3, seed=k3 + 300, rows=only)
    got = host_backward(aa_shim, sc, k3, up, pose)
    ref, st, s, gc2 = oracle_backward(sc, k3, up)
    keep = st["keep"]
    flag = s["near"] | (rel_tol(s) > 1e-3)  # ill-conditioned or at the clamp: bounded separately below
    for name in ("pws", "scales", "rots", "shs"):
        g = got[name].astype(np.float64)
        scale = np.abs(ref[name]).max()
        e = np.abs(g - ref[name])[~flag].max() / scale
        assert e < 3e-5, (name, e)
        if flag.any():
            assert np.isfinite(g[flag]).all()
    e = np.abs(got["alphas"] - ref["alphas"]) / np.maximum(np.abs(ref["alphas"]), 1e-30)
    assert np.all((e <= rel_tol(s)) | s["near"])
    # dL/dalpha_eff alone moves the geometry of kept, unclamped rows
    live = only[keep[only] & ~s["clamped"][only]]
    assert len(live) > 10 and np.all(np.abs(got["scales"][live]).sum(1) > 0)
    # clamped rows: the non-AA geometry gradient and 0.005 galpha for alpha
    z = rows["zero"]
    assert np.all(s["clamped"][z]) and not gc2[z].any()
    rho_min = np.float32(np.sqrt(np.float32(2.5e-5)))
    assert np.array_equal(got["alphas"][z], (rho_min * up[4][z]).astype(np.float32))
    # culled rows: dL/dalpha = dL/dalpha_eff
    c = rows["culled"]
    assert np.array_equal(got["alphas"][c], up[4][c])
    if pose:
        for col in range(15):
            sref = np.abs(ref["cam"][:, col]).max()
            if sref == 0:
                continue
            e = np.abs(got["cam"][~flag, col].astype(np.float64) - ref["cam"][~flag, col]).max() / sref
            assert e <= 3e-5, (col, e)
        # the per-Gaussian outputs are those of the form without the camera, bit for bit
        plain = host_backward(aa_shim, sc, k3, up, False)
        for k in ("pws", "shs", "scales", "rots", "alphas"):
            assert np.array_equal(got[k].view(np.uint32), plain[k].view(np.uint32)), k


# ---------------------------------------------------------------- the property
def _coverage(sc, scale_down, aa):
    """mean opacity coverage (1 - final transmittance) of the oracle renderer at 1/scale_down of the
    frame, with or without the compensation"""
    w, h = W // scale_down, H // scale_down
    fx, fy, cx, cy = (sc[k] / scale_down for k in ("fx", "fy", "cx", "cy"))
    st = oaa.stages(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], fx, fy, cx, cy,
                    w, h)
    al = sc["alphas"] * (oaa.scale(st["c2"], st["keep"])["rho"] if aa else 1.0)
    out = orc.splat(h, w, st["us"], st["ci"], al, st["depths"].copy(), st["col"], st["areas"].copy())
    return float((1.0 - out["final_tau"]).mean())


def test_coverage_is_scale_consistent_with_aa():
    """A field of Gaussians about one pixel across at full resolution: drawn at a quarter of the
    resolution, without the compensation every one of them still becomes a ~0.55 px blob at full
    opacity and the frame's coverage balloons; with it the coverage stays much closer.  Measured on
    this scene (oracle, fp64): mean coverage 0.324 -> 0.696 (x2.15) without, 0.283 -> 0.279 (x0.99)
    with; the test asks for x1.5 without and half the log-ratio with."""
    sc = _scene(4000, 1, seed=5, rotate=False)
    rng = np.random.default_rng(6)
    N = len(sc["pws"])
    sc["pws"][:, 2] = np.abs(sc["pws"][:, 2]) + 1.0  # nothing culled
    z = sc["pws"][:, 2] + sc["tcw"][2]
    sc["scales"] = (np.full((N, 3), 1.0, np.float32) * (z / sc["fx"])[:, None] *
                    rng.uniform(0.5, 1.5, (N, 1))).astype(np.float32)
    sc["alphas"] = rng.uniform(0.3, 0.9, N).astype(np.float32)
    ratio = {aa: _coverage(sc, 4, aa) / _coverage(sc, 1, aa) for aa in (False, True)}
    assert ratio[False] > 1.5, ratio
    assert abs(np.log(ratio[True])) < 0.5 * abs(np.log(ratio[False])), ratio


# ---------------------------------------------------------------- the sm_90a binary
def test_aa_kernels_are_sm90a_without_spills():
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    r = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True)
    assert r.returncode == 0
    bwd, fwd = {}, {}
    for name, usage in re.findall(r"Function (_ZN3gsb16k_preprocess_(?:fwd|bwd)\S+):\s*\n\s*(REG:.*)", r.stdout):
        t = re.search(r"ILi(\d+)((?:ELb\d)+)E", name)
        flags = tuple(re.findall(r"Lb(\d)", t.group(2)))
        if "fwd" in name:
            fwd[(t.group(1),) + flags] = usage
        else:
            bwd[(t.group(1),) + flags] = usage
    ks = ("1", "4", "9", "16")
    assert {k for k in fwd if k[-1] == "1"} == {(k, "1") for k in ks}
    # AA: with MOM, never with PUSH -> 4 forms (DEPTH x POSE) per SH degree
    assert {k for k in bwd if k[-1] == "1"} == {(k, "0", "1", d, p, "1") for k in ks for d in "01" for p in "01"}
    for t, usage in list(fwd.items()) + list(bwd.items()):
        if t[-1] == "1":  # no spills; at most the 8-byte frame of the slow-path division calls that
            # the parent's K3 = 9 and 16 RGB-D backward forms have too
            assert "LOCAL:0 " in usage and re.search(r"STACK:[08] ", usage), (t, usage)
