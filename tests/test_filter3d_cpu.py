"""CPU checks of the Mip-Splatting 3D smoothing filter: the fp64 oracle (oracle/filter3d_oracle.py)
against central differences, alone and through the whole rendered loss; the host build of the
filter math (pg_fused_math.h through tests/host_shim/filter3d_host.cpp) against the oracle on
constructed boundary cameras, random camera sets and edge rows; the properties the filter exists
for; and the kernels in the sm_90a binary."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import filter3d_oracle as of3
from oracle import oracle as orc
from easygaussiansplatting_b200.scene import synthetic_scene, upstream_gradient

from test_fused_math_cpu import _p
from test_oracle_fd import _forward

HERE = os.path.dirname(os.path.abspath(__file__))
F3_SO = os.path.join(HERE, "host_shim", "_build", "libfilter3d_host.so")


@pytest.fixture(scope="module")
def f3_shim():
    src = os.path.join(HERE, "host_shim", "filter3d_host.cpp")
    hdr = os.path.join(HERE, "..", "easygaussiansplatting_b200", "csrc", "pg_fused_math.h")
    os.makedirs(os.path.dirname(F3_SO), exist_ok=True)
    if not os.path.exists(F3_SO) or os.path.getmtime(F3_SO) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", F3_SO, src],
                       check=True)
    return C.CDLL(F3_SO)


# ---------------------------------------------------------------- shared scenes (also the GPU tests')
def camera_row(Rcw, tcw, fx, fy, cx, cy, W, H):
    row = np.zeros(20, np.float32)
    row[:9] = np.asarray(Rcw, np.float32).reshape(-1)
    row[9:12] = np.asarray(tcw, np.float32).reshape(-1)
    row[12:18] = [fx, fy, cx, cy, W, H]
    return row


def look_at(eye, target):
    """-> (Rcw, tcw) of a camera at `eye` whose optical axis (+z) points at `target`"""
    eye, target = np.asarray(eye, np.float64), np.asarray(target, np.float64)
    z = target - eye
    z /= np.linalg.norm(z)
    x = np.cross(z, [0.0, 1.0, 0.0])
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])
    return R, -R @ eye


def ring_table(C, seed, W=320, H=240):
    """C cameras on a ring of radius 4-8 around the unit box, looking near its centre, with fx in
    [150, 450] (different for every camera) and principal points off the frame centre"""
    rng = np.random.default_rng(seed)
    rows = []
    for k in range(C):
        a = 2 * np.pi * (k + rng.uniform()) / max(C, 1)
        r = rng.uniform(4.0, 8.0)
        eye = [r * np.cos(a), rng.uniform(-1.0, 1.0), r * np.sin(a)]
        R, t = look_at(eye, rng.uniform(-0.5, 0.5, 3))
        fx = rng.uniform(150.0, 450.0)
        rows.append(camera_row(R, t, fx, fx * rng.uniform(0.9, 1.1), W / 2 + rng.uniform(-20, 20),
                               H / 2 + rng.uniform(-20, 20), W, H))
    return np.stack(rows) if rows else np.zeros((0, 20), np.float32)


def box_points(N, seed, unseen=0.05):
    """N points in [-2, 2]^3; a fraction `unseen` far above the ring, where no camera looks"""
    rng = np.random.default_rng(seed)
    p = rng.uniform(-2.0, 2.0, (N, 3))
    far = rng.uniform(size=N) < unseen
    p[far] = [0.0, 500.0, 0.0] + rng.uniform(-1, 1, (int(far.sum()), 3))
    return p.astype(np.float32), far


def host_filter(lib, pws, table, variance=0.2):
    N = len(pws)
    out = np.empty(N, np.float32)
    lib.filter3d_host(N, _p(pws), len(table), _p(np.ascontiguousarray(table, np.float32)) if len(table) else None,
                      C.c_float(variance), _p(out))
    return out


def host_depth(lib, pws, table):
    N = len(pws)
    out = np.empty(N, np.float32)
    lib.filter3d_depth_host(N, _p(pws), len(table), _p(np.ascontiguousarray(table, np.float32)), _p(out))
    return out


def host_apply(lib, s, a, f):
    N = len(a)
    sf, af = np.empty((N, 3), np.float32), np.empty(N, np.float32)
    lib.filter3d_apply_host(N, _p(s), _p(a), _p(f), _p(sf), _p(af))
    return sf, af


def host_backward(lib, s, a, f, gsf, gaf):
    N = len(a)
    gs, ga = np.empty((N, 3), np.float32), np.empty(N, np.float32)
    lib.filter3d_backward_host(N, _p(s), _p(a), _p(f), _p(gsf), _p(gaf), _p(gs), _p(ga))
    return gs, ga


def edge_rows(seed, n=4000):
    """(scales, alphas, filter) with the edge rows at the head: 0-7 f = 0, 8-15 s = 0 (one axis or
    all), 16-23 needles, 24-31 f >> s, 32-39 f << s; the rest random around f ~ s"""
    rng = np.random.default_rng(seed)
    s = np.exp(rng.uniform(-6, 0, (n, 3))).astype(np.float32)
    a = rng.uniform(0.01, 1.0, n).astype(np.float32)
    f = (np.exp(rng.uniform(-6, 0, n))).astype(np.float32)
    f[0:8] = 0.0
    s[8:12, 0] = 0.0
    s[12:16] = 0.0
    s[16:24] = np.array([0.5, 1e-4, 1e-4], np.float32)
    f[24:32] = s[24:32].max(1) * 1e3
    f[32:40] = s[32:40].min(1) * 1e-3
    s[0:2] = 0.0  # s = f = 0
    rows = dict(zero_f=np.arange(8), zero_s=np.arange(8, 16), needle=np.arange(16, 24), big_f=np.arange(24, 32),
                small_f=np.arange(32, 40))
    return s, a, f, rows


# ---------------------------------------------------------------- the oracle itself
def test_oracle_apply_backward_vs_central_differences():
    """L = sum w_s . s' + w_a alpha' (random weights): the oracle backward against central
    differences of the oracle apply in every scale and the opacity, in fp64"""
    s, a, f, _ = edge_rows(3, n=300)
    s, a, f = s[40:].astype(np.float64), a[40:].astype(np.float64), f[40:].astype(np.float64)
    rng = np.random.default_rng(4)
    ws, wa = rng.normal(size=s.shape), rng.normal(size=a.shape)
    gs, ga = of3.backward(s, a, f, ws, wa)
    L = lambda s_, a_: (of3.apply(s_, a_, f)[0] * ws).sum(1) + of3.apply(s_, a_, f)[1] * wa
    for j in range(3):
        h = 1e-6 * s[:, j]
        sp, sm = s.copy(), s.copy()
        sp[:, j] += h; sm[:, j] -= h
        fd = (L(sp, a) - L(sm, a)) / (2 * h)
        assert np.allclose(gs[:, j], fd, rtol=1e-6, atol=1e-9 * np.abs(fd).max()), j
    h = 1e-6 * a
    fd = (L(s, a + h) - L(s, a - h)) / (2 * h)
    assert np.allclose(ga, fd, rtol=1e-6, atol=1e-9 * np.abs(fd).max())


def test_oracle_chain_vs_central_differences():
    """The whole oracle loss sum(image * dl) of a frame rendered from s', alpha': the existing
    chain_backward on s', alpha' and then the filter backward, against central differences in the
    unfiltered scales and alphas (the forward is only piecewise smooth: test_oracle_fd's three step
    sizes, a parameter passes when one of them reproduces the analytic value)"""
    N, W, H = 160, 64, 48
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=13)
    sc = {k: (np.asarray(v, dtype=np.float64) if isinstance(v, np.ndarray) else v) for k, v in sc.items()}
    table = camera_row(sc["Rcw"], sc["tcw"], sc["fx"], sc["fy"], sc["cx"], sc["cy"], W, H)[None]
    filt = of3.filter3d(sc["pws"], table)["filter"]
    assert (filt > 0).all()
    dl = upstream_gradient(W, H, 5).astype(np.float64) * (3.0 * W * H)
    s0, a0 = sc["scales"].copy(), sc["alphas"].copy()

    def loss(s, a):
        sf, af, _ = of3.apply(s, a, filt)
        return _forward(dict(sc, scales=sf, alphas=af), W, H, dl)

    lval, (us, ci, col, fwd, Ju, J3r, J3s, J2c, J2p, Jcs, Jcp, Jci) = loss(s0, a0)
    _, af, _ = of3.apply(s0, a0, filt)
    g4 = orc.splat_backward(H, W, us, ci, af, col, fwd, dl)
    chain = orc.chain_backward(sc["Rcw"], *g4, Ju, J3r, J3s, J2c, J2p, Jcs, Jcp, Jci)
    gs, ga = of3.backward(s0, a0, filt, chain["scales"], np.asarray(g4[2]).reshape(-1))
    used = np.unique(fwd["gsid"])
    rng = np.random.default_rng(6)
    good = checked = 0
    for _ in range(70):
        i = int(rng.choice(used))
        j = int(rng.integers(4))  # 0-2 a scale, 3 the opacity
        an = float(gs[i, j] if j < 3 else ga[i])
        x0 = float(s0[i, j] if j < 3 else a0[i])
        checked += 1
        for rel in (2e-3, 5e-4, 1.5e-4):
            h = rel * max(abs(x0), 0.05 if j == 3 else 1e-3)
            lp, lm = [], []
            for sign, acc in ((1, lp), (-1, lm)):
                s, a = s0.copy(), a0.copy()
                if j < 3:
                    s[i, j] = x0 + sign * h
                else:
                    a[i] = x0 + sign * h
                acc.append(loss(s, a)[0])
            fd = (lp[0] - lm[0]) / (2 * h)
            if abs(fd - an) <= 1e-2 * max(abs(fd), abs(an)) + 1e-6 * abs(lval):
                good += 1
                break
    assert good >= int(0.85 * checked), "only %d of %d finite differences agree" % (good, checked)


# ---------------------------------------------------------------- host build vs oracle
def test_host_visibility_on_boundary_cameras(f3_shim):
    """Constructed so that z and u land exactly on the bounds (R = I, t = 0, fx = fy = 1, cx = cy = 0,
    z = 0.25: u = 4 x exactly): on a bound is seen, one ulp outside is not; z = 0.2f is kept, the
    next float below is culled.  The oracle flags every one of these rows."""
    W, H = np.float32(200.0), np.float32(120.0)
    cam = camera_row(np.eye(3), np.zeros(3), 1.0, 1.0, 0.0, 0.0, W, H)
    lo_x, hi_x = np.float32(-of3.MARGIN * W), np.float32(of3.HI * W)
    lo_y, hi_y = np.float32(-of3.MARGIN * H), np.float32(of3.HI * H)
    q = np.float32(0.25)
    four = lambda v: np.float32(v / np.float32(4.0))
    out = lambda v, d: np.nextafter(four(v), np.float32(d))
    inner_y = four(np.float32(10.0))
    pts, want = [], []
    for bx in (lo_x, hi_x):
        pts.append([four(bx), inner_y, q]); want.append(True)
        pts.append([out(bx, -np.inf if bx < 0 else np.inf), inner_y, q]); want.append(False)
    for by in (lo_y, hi_y):
        pts.append([four(np.float32(10.0)), four(by), q]); want.append(True)
        pts.append([four(np.float32(10.0)), out(by, -np.inf if by < 0 else np.inf), q]); want.append(False)
    z0 = np.float32(0.2)
    cam_z = camera_row(np.eye(3), np.zeros(3), 1.0, 1.0, 0.0, 0.0, W, H)
    pts_z = np.array([[0.0, 0.0, z0], [0.0, 0.0, np.nextafter(z0, np.float32(0))]], np.float32)
    pws = np.array(pts, np.float32)
    d = host_depth(f3_shim, pws, cam[None])
    assert list(d > 0) == want, (d, want)
    assert np.array_equal(d[np.array(want)], pws[np.array(want), 2])
    dz = host_depth(f3_shim, pts_z, cam_z[None])
    assert dz[0] == z0 and dz[1] == 0.0
    seen, z32, flag = of3.visibility(pws, cam)
    assert flag.all() and list(seen) == want
    seen_z, _, flag_z = of3.visibility(pts_z, cam_z)
    assert flag_z.all() and list(seen_z) == [True, False]


@pytest.mark.parametrize("C", [1, 7, 64, 129])
def test_host_filter_matches_oracle(f3_shim, C):
    """random camera rings: d_i bit for bit on every unflagged row (variance = fmax^2 with fmax a
    power of two makes the filter value d itself), the filter to 1e-6 relative at variance 0.2"""
    pws, far = box_points(3000, seed=C)
    table = ring_table(C, seed=100 + C)
    table[0, 12] = 512.0  # the largest fx, a power of two
    ref = of3.filter3d(pws, table)
    assert ref["seen"].sum() > 2000 and not ref["seen"][far].any()
    assert ref["flagged"].sum() <= 3
    ok = ~ref["flagged"]
    got = host_filter(f3_shim, pws, table, variance=512.0 ** 2)
    assert np.array_equal(got[ok], ref["d"][ok].astype(np.float32))
    got = host_filter(f3_shim, pws, table).astype(np.float64)
    assert np.all(np.abs(got - ref["filter"])[ok] <= 1e-6 * ref["filter"][ok])


def test_host_filter_nothing_seen(f3_shim):
    """no row seen -> every filter value 0 (also with no camera at all, and with no fx > 0)"""
    pws = (np.random.default_rng(1).uniform(-1, 1, (100, 3)) + [0, 500, 0]).astype(np.float32)
    table = ring_table(5, seed=2)
    assert not host_filter(f3_shim, pws, table).any()
    assert not of3.filter3d(pws, table)["filter"].any()
    assert not host_filter(f3_shim, pws, table[:0]).any()
    # seen rows but no camera with fx > 0: zeros, not d / 0
    seen_pws, _ = box_points(500, seed=3)
    bad = table.copy()
    bad[:, 12] = -np.abs(bad[:, 12])
    assert of3.filter3d(seen_pws, bad)["dmax"] > 0
    assert not host_filter(f3_shim, seen_pws, bad).any() and not of3.filter3d(seen_pws, bad)["filter"].any()


def test_host_apply_backward_edge_rows(f3_shim):
    s, a, f, rows = edge_rows(9)
    sf, af = host_apply(f3_shim, s, a, f)
    rsf, raf, _ = of3.apply(s, a, f)
    z = rows["zero_f"]  # f == 0: both pass through bit for bit (s = f = 0 included)
    assert np.array_equal(sf[z].view(np.uint32), s[z].view(np.uint32))
    assert np.array_equal(af[z].view(np.uint32), a[z].view(np.uint32))
    assert np.all(np.abs(sf - rsf) <= 4e-7 * rsf)
    assert np.all(np.abs(af - raf) <= 1e-6 * raf + 1e-30)
    zs = rows["zero_s"]  # s = 0 with f > 0: s' = f on that axis, alpha' = 0
    assert np.all(af[zs] == 0.0) and np.all(sf[zs][s[zs] == 0] == np.broadcast_to(f[zs, None], (8, 3))[s[zs] == 0])
    rng = np.random.default_rng(10)
    gsf = rng.normal(size=s.shape).astype(np.float32)
    gaf = rng.normal(size=a.shape).astype(np.float32)
    gs, ga = host_backward(f3_shim, s, a, f, gsf, gaf)
    rgs, rga = of3.backward(s, a, f, gsf, gaf)
    assert np.array_equal(gs[z].view(np.uint32), gsf[z].view(np.uint32))
    assert np.array_equal(ga[z].view(np.uint32), gaf[z].view(np.uint32))
    assert np.isfinite(gs).all() and np.isfinite(ga).all()
    # each term is within a few ulp of its magnitude: bound by the sum of the terms' magnitudes
    _, _, t = of3.apply(s, a, f)
    mag = np.abs(gsf) * t + np.abs(rgs - gsf * t) + 1e-30
    assert np.all(np.abs(gs - rgs) <= 2e-6 * mag)
    assert np.all(np.abs(ga - rga) <= 1e-6 * np.abs(rga) + 1e-30)
    # in place: the outputs may be the inputs
    gs2, ga2 = gsf.copy(), gaf.copy()
    f3_shim.filter3d_backward_host(len(a), _p(s), _p(a), _p(f), _p(gs2), _p(ga2), _p(gs2), _p(ga2))
    assert np.array_equal(gs2, gs) and np.array_equal(ga2, ga)


# ---------------------------------------------------------------- the properties
def test_mass_is_preserved():
    s, a, f, _ = edge_rows(11)
    s, a, f = s.astype(np.float64), a.astype(np.float64), f.astype(np.float64)
    sf, af, _ = of3.apply(s, a, f)
    m0, m1 = a * s.prod(1), af * sf.prod(1)
    assert np.all(np.abs(m1 - m0) <= 1e-12 * np.maximum(m0, 1e-300))


def test_filtered_std_projects_to_at_least_sqrt_variance_pixels():
    """at a camera with fx = f_max placed at depth d_i, the smallest filtered std covers >= sqrt(variance) px"""
    pws, _ = box_points(2000, seed=4)
    table = ring_table(9, seed=5)
    ref = of3.filter3d(pws, table, variance=0.2)
    s = np.exp(np.random.default_rng(6).uniform(-9, -1, (2000, 3)))
    sf, _, _ = of3.apply(s, np.ones(2000), ref["filter"])
    px = sf.min(1) * ref["fmax"] / ref["d"]
    assert np.all(px >= np.sqrt(0.2) * (1 - 1e-12))


def _coverage(pws, scales, alphas, fx, W, H):
    """mean opacity coverage (1 - final transmittance) of the oracle renderer, camera at the origin"""
    N = len(pws)
    rots = np.tile(np.array([1, 0, 0, 0], np.float32), (N, 1))
    shs = np.zeros((N, 3), np.float32)
    us, pcs, depths, _ = orc.project(pws, np.eye(3), np.zeros(3), fx, fx, W / 2, H / 2)
    d32 = depths.astype(np.float32)
    c3 = orc.compute_cov3d(rots, scales, d32, calc_J=False)[0]
    c2 = orc.compute_cov2d(c3, pcs, np.eye(3), d32, fx, fx, W, H, calc_J=False)[0]
    col = orc.sh2color(shs, pws, np.zeros(3), calc_J=False)[0]
    ci, areas = orc.inverse_cov2d(c2, d32, calc_J=False)
    out = orc.splat(H, W, us, ci, alphas, d32, col, areas)
    return float((1.0 - out["final_tau"]).mean())


def test_zoom_coverage_is_closer_with_the_filter():
    """A field of sub-pixel Gaussians (std 0.2-0.3 px at the training camera): zoomed in 4x, the
    unfiltered field erodes (each Gaussian drawn at full opacity was a 0.6 px blob in training and is
    a thin 1 px one now) and its coverage drops; the filtered one keeps much closer to what was
    trained.  Measured (oracle, fp64): coverage ratio zoom / training 0.442 unfiltered, 0.564
    filtered; the test asks that the filtered log-ratio be at most 0.8 of the unfiltered one."""
    rng = np.random.default_rng(8)
    N, W, H, fx = 30000, 160, 120, 200.0
    z = rng.uniform(4.0, 6.0, N)
    u, v = rng.uniform(0, W, N), rng.uniform(0, H, N)
    pws = np.stack([(u - W / 2) * z / fx, (v - H / 2) * z / fx, z], 1).astype(np.float32)
    scales = ((z / fx)[:, None] * rng.uniform(0.2, 0.3, (N, 3))).astype(np.float32)
    alphas = rng.uniform(0.3, 0.9, N).astype(np.float32)
    table = camera_row(np.eye(3), np.zeros(3), fx, fx, W / 2, H / 2, W, H)[None]
    filt = of3.filter3d(pws, table)["filter"]
    sf, af, _ = of3.apply(scales, alphas, filt)
    ratio = {}
    for name, s, a in (("plain", scales, alphas), ("filtered", sf.astype(np.float32), af.astype(np.float32))):
        ratio[name] = _coverage(pws, s, a, 4 * fx, W, H) / _coverage(pws, s, a, fx, W, H)
    assert ratio["plain"] < 0.5, ratio
    assert abs(np.log(ratio["filtered"])) <= 0.8 * abs(np.log(ratio["plain"])), ratio


# ---------------------------------------------------------------- the sm_90a binary
def test_filter3d_kernels_are_sm90a_without_spills():
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    r = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True)
    assert r.returncode == 0
    found = dict(re.findall(r"Function _ZN3gsb\d+(k_filter3d_\w+?)E\S*:\s*\n\s*(REG:.*)", r.stdout))
    assert set(found) == {"k_filter3d_depth", "k_filter3d_finish", "k_filter3d_apply", "k_filter3d_bwd"}, found
    for name, usage in found.items():
        assert "LOCAL:0 " in usage and "STACK:0 " in usage, (name, usage)
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert re.search(r"Function : _ZN3gsb16k_filter3d_depth", sass) and "sm_90a" in sass
