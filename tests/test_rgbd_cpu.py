"""CPU checks of RGB-D rendering (depth D = sum w z and opacity A = sum w with the image's
compositing weights): the fp64 oracle's RGB-D pair against its colour pair and against central
finite differences of the whole chain, the depth term of the fused per-Gaussian backward
(pg_fused_math.h through the host shim) against the oracle chain, and the two RGB-D rasterizers
in the sm_90a binary."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import oracle as orc
from oracle import rgbd_oracle as orgbd
from easygaussiansplatting_b200.scene import synthetic_scene, upstream_gradient

from test_fused_math_cpu import _oracle_stages, _p, _scene, shim  # noqa: F401  (shim is a fixture)

HERE = os.path.dirname(os.path.abspath(__file__))
DEPTH_SO = os.path.join(HERE, "host_shim", "_build", "libfused_depth_host.so")


@pytest.fixture(scope="module")
def depth_shim():
    """tests/host_shim/fused_depth_host.cpp: backward_one with the depth gradient, host build"""
    src = os.path.join(HERE, "host_shim", "fused_depth_host.cpp")
    hdr = os.path.join(HERE, "..", "easygaussiansplatting_b200", "csrc", "pg_fused_math.h")
    os.makedirs(os.path.dirname(DEPTH_SO), exist_ok=True)
    if not os.path.exists(DEPTH_SO) or os.path.getmtime(DEPTH_SO) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", DEPTH_SO, src],
                       check=True)
    return C.CDLL(DEPTH_SO)


def _stages(sc, W, H):
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    us, pcs, depths, Ju = orc.project(sc["pws"], sc["Rcw"], sc["tcw"], sc["fx"], sc["fy"], sc["cx"], sc["cy"])
    d32 = f32(depths)
    c3, J3r, J3s = orc.compute_cov3d(sc["rots"], sc["scales"], d32)
    c2, J2c, J2p = orc.compute_cov2d(c3, pcs, sc["Rcw"], d32, sc["fx"], sc["fy"], W, H)
    col, Jcs, Jcp = orc.sh2color(sc["shs"], sc["pws"], sc["twc"])
    ci, areas, Jci = orc.inverse_cov2d(c2, d32)
    return us, ci, col, d32, areas, (Ju, J3r, J3s, J2c, J2p, Jcs, Jcp, Jci)


def _scene64(N, W, H, seed, sh_dim=12):
    sc = synthetic_scene(N, W, H, sh_dim=sh_dim, seed=seed)
    return {k: (np.asarray(v, dtype=np.float64) if isinstance(v, np.ndarray) else v) for k, v in sc.items()}


def test_rgbd_oracle_reduces_to_the_colour_oracle():
    N, W, H = 600, 97, 61
    sc = _scene64(N, W, H, seed=3)
    us, ci, col, d32, areas, _ = _stages(sc, W, H)
    al = sc["alphas"]
    f = orc.splat(H, W, us, ci, al, d32.copy(), col, areas.copy())
    g = orgbd.splat_rgbd(H, W, us, ci, al, d32.copy(), col, areas.copy())
    for k in ("image", "contrib", "final_tau", "ranges", "gsid", "ambiguous"):
        assert np.array_equal(f[k], g[k]), k
    # opacity is what the transmittance lost, on every pixel of a tile with patches
    T = ((W + 15) // 16) * ((H + 15) // 16)
    has = (g["ranges"][:, 1] > g["ranges"][:, 0]).reshape((H + 15) // 16, (W + 15) // 16)
    drawn = np.kron(has, np.ones((16, 16), bool))[:H, :W]
    assert T == has.size and drawn.any()
    assert np.abs(g["alpha"] - (1.0 - g["final_tau"]))[drawn].max() <= 1e-12
    assert not g["alpha"][~drawn].any() and not g["depth"][~drawn].any()
    # D / A lies between the nearest and farthest drawn depth
    m = g["alpha"] > 1e-3
    zs = g["z"][np.unique(g["gsid"])]
    ed = g["depth"][m] / g["alpha"][m]
    assert ed.min() >= zs.min() * (1 - 1e-12) and ed.max() <= zs.max() * (1 + 1e-12)
    # the backward with dL/dD = dL/dA = 0 is the colour backward, and dL/dz = 0
    dl = upstream_gradient(W, H, 3).astype(np.float64) * (3.0 * W * H)
    zero = np.zeros((H, W), np.float32)
    b4 = orc.splat_backward(H, W, us, ci, al, col, f, dl)
    b5 = orgbd.splat_backward_rgbd(H, W, us, ci, al, col, g["z"], g, dl, zero, zero)
    for a, b in zip(b4, b5[:4]):  # (the oracle sums with OpenMP atomics: order-level differences)
        assert np.abs(a - b).max() <= 1e-12 * np.abs(a).max()
    assert not b5[4].any()


def _loss_rgbd(sc, W, H, G):
    us, ci, col, d32, areas, J = _stages(sc, W, H)
    fwd = orgbd.splat_rgbd(H, W, us, ci, sc["alphas"], d32, col, areas)
    loss = float((fwd["image"] * G[0]).sum() + (fwd["depth"] * G[1]).sum() + (fwd["alpha"] * G[2]).sum())
    return loss, (us, ci, col, fwd, J)


def test_rgbd_full_chain_gradient_vs_central_differences():
    """L = <G1, image> + <G2, D> + <G3, A>: the oracle's analytic gradient (splat_backward_rgbd +
    Jacobian chain + the depth term dL/dz Rcw[2,:]) against central differences of its forward,
    for pws (through u, the conic and z), scales, rots, shs and alphas"""
    N, W, H = 160, 64, 48
    sc = _scene64(N, W, H, seed=11)
    rng = np.random.default_rng(4)
    G = (upstream_gradient(W, H, 3).astype(np.float64) * (3.0 * W * H),
         rng.normal(size=(H, W)) * 0.3, rng.normal(size=(H, W)))
    loss, (us, ci, col, fwd, J) = _loss_rgbd(sc, W, H, G)
    b5 = orgbd.splat_backward_rgbd(H, W, us, ci, sc["alphas"], col, fwd["z"], fwd, G[0], G[1], G[2])
    chain = orc.chain_backward(sc["Rcw"], *b5[:4], *J)
    dpws = chain["pws"] + orgbd.chain_depth(sc["Rcw"], b5[4], fwd["z"])
    assert np.abs(orgbd.chain_depth(sc["Rcw"], b5[4], fwd["z"])).max() > 1e-3 * np.abs(dpws).max()
    grads = {"pws": dpws, "scales": chain["scales"], "rots": chain["rots"], "shs": chain["shs"],
             "alphas": np.asarray(b5[2]).reshape(-1)}
    used = np.unique(fwd["gsid"])
    picks = []
    while len(picks) < 80:
        name = ("pws", "pws", "scales", "rots", "shs", "alphas")[rng.integers(6)]
        i = int(rng.choice(used))
        j = 0 if name == "alphas" else int(rng.integers(sc[name].shape[1]))
        picks.append((name, i, j))
    good = 0
    for name, i, j in picks:
        x = sc[name]
        idx = (i,) if name == "alphas" else (i, j)
        x0 = float(x[idx])
        an = float(grads[name][i] if name == "alphas" else grads[name].reshape(N, -1)[i, j])
        # piecewise smooth forward, fp32-rounded stage inputs: three step sizes (test_oracle_fd.py)
        for rel in (2e-3, 5e-4, 1.5e-4):
            h = rel * max(abs(x0), 0.05)
            x[idx] = x0 + h
            lp = _loss_rgbd(sc, W, H, G)[0]
            x[idx] = x0 - h
            lm = _loss_rgbd(sc, W, H, G)[0]
            x[idx] = x0
            fd = (lp - lm) / (2 * h)
            if abs(fd - an) <= 1e-2 * max(abs(fd), abs(an)) + 1e-6 * abs(loss):
                good += 1
                break
    assert good >= int(0.85 * len(picks)), "only %d of %d finite differences agree" % (good, len(picks))


@pytest.mark.parametrize("k3", [1, 4, 9, 16])
def test_fused_backward_depth_term_matches_oracle_chain(shim, depth_shim, k3):  # noqa: F811
    W, H, N = 320, 240, 3000
    sc = _scene(N, k3, seed=30 + k3)
    o = _oracle_stages(sc, W, H)
    rng = np.random.default_rng(k3 + 100)
    gu = rng.normal(size=(N, 1, 2)).astype(np.float32)
    gci = rng.normal(size=(N, 1, 3)).astype(np.float32) * 10
    gcol = rng.normal(size=(N, 1, 3)).astype(np.float32)
    gz = rng.normal(size=N).astype(np.float32)
    gz[N // 2:N // 2 + 50] *= 1e3
    keep = o["depths"] > 0
    # a Gaussian with only a depth gradient must not be skipped by the zero-gradient gate
    only = np.flatnonzero(keep)[:40]
    gu[only] = 0; gci[only] = 0; gcol[only] = 0
    gu[~keep] = 0; gci[~keep] = 0; gcol[~keep] = 0
    gal = np.zeros((N, 1, 1), np.float32)
    ref = orc.chain_backward(sc["Rcw"], gu, gci, gal, gcol, *o["J"])
    ref_pws = ref["pws"] + orgbd.chain_depth(sc["Rcw"], gz, o["depths"])
    out = {k: np.empty(s, np.float32) for k, s in (("pws", (N, 3)), ("shs", (N, 3 * k3)), ("scales", (N, 3)),
                                                   ("rots", (N, 4)))}
    rc = depth_shim.fused_backward_depth_host(N, k3, _p(sc["pws"]), _p(sc["rots"]), _p(sc["scales"]), _p(sc["shs"]),
                                        _p(sc["Rcw"]), _p(sc["tcw"]), _p(sc["twc"]), C.c_float(sc["fx"]),
                                        C.c_float(sc["fy"]), C.c_float(sc["cx"]), C.c_float(sc["cy"]), C.c_float(W),
                                        C.c_float(H), _p(gu), _p(gci), _p(gcol), _p(gz), _p(out["pws"]),
                                        _p(out["shs"]), _p(out["scales"]), _p(out["rots"]))
    assert rc == 0
    for name, want in (("pws", ref_pws), ("shs", ref["shs"]), ("scales", ref["scales"]), ("rots", ref["rots"])):
        e = np.abs(out[name].astype(np.float64) - want).max() / np.abs(want).max()
        assert e < 2e-5, (name, e)
    e = np.abs(out["pws"][only] - ref_pws[only]).max() / np.abs(ref_pws[only]).max()
    assert e < 1e-6 and np.abs(out["pws"][only]).min() > 0
    assert (~keep).any() and not out["pws"][~keep].any()  # culled (z < 0.2): no depth gradient either
    # gz = 0 reproduces the colour-only backward bit for bit
    z = np.zeros(N, np.float32)
    out0 = {k: np.empty_like(v) for k, v in out.items()}
    col0 = {k: np.empty_like(v) for k, v in out.items()}
    args = [_p(sc["pws"]), _p(sc["rots"]), _p(sc["scales"]), _p(sc["shs"]), _p(sc["Rcw"]), _p(sc["tcw"]),
            _p(sc["twc"]), C.c_float(sc["fx"]), C.c_float(sc["fy"]), C.c_float(sc["cx"]), C.c_float(sc["cy"]),
            C.c_float(W), C.c_float(H), _p(gu), _p(gci), _p(gcol)]
    depth_shim.fused_backward_depth_host(N, k3, *args, _p(z), *[_p(out0[k]) for k in ("pws", "shs", "scales", "rots")])
    shim.fused_backward_host(N, k3, *args, *[_p(col0[k]) for k in ("pws", "shs", "scales", "rots")])
    for k in out0:
        assert np.array_equal(out0[k], col0[k]), k


def test_rgbd_rasterizers_are_sm90a_with_cp_async_record_gather():
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    r = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True)
    funcs = re.split(r"\n\s*Function : ", r.stdout)
    for name in ("k_draw_rgbd", "k_draw_bwd_rgbd"):
        body = [f for f in funcs if f.startswith("_ZN3gsb%d%sE" % (len(name), name))]
        assert len(body) == 1, name
        for op in ("LDGSTS.E.BYPASS.128", "LDGDEPBAR", "DEPBAR.LE", "MUFU.EX2"):
            assert op in body[0], "%s: %s missing" % (name, op)
    lib = _lib.load()
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    assert names.index("draw") == 11 and names.index("draw_backward") == 12
    assert names[-2:] == ["draw_rgbd", "draw_backward_rgbd"]
