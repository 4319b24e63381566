"""CPU checks of feature rendering (per-Gaussian features composited with the image's weights):
the fp64 feature oracle against the colour and RGB-D oracles it is built from, its linearity in the
channels, its gradients against central differences, and the C ABI / sm_90a binary of the two
feature rasterizers and the density row rebuild."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest

from oracle import feature_oracle as ofe
from oracle import oracle as orc
from oracle import rgbd_oracle as orgbd
from easygaussiansplatting_b200.scene import upstream_gradient

from test_host_cpu import header_symbols
from test_rgbd_cpu import _scene64, _stages

W, H, N = 97, 61, 600


@pytest.fixture
def serial():
    """the oracle's rasterizer backward sums with OpenMP atomics: one thread for bit-level equality"""
    n0 = orc.num_threads()
    orc.set_num_threads(1)
    yield
    orc.set_num_threads(n0)


def _frame(seed=3, n=N, w=W, h=H):
    sc = _scene64(n, w, h, seed=seed)
    us, ci, col, d32, areas, _ = _stages(sc, w, h)
    return sc, us, ci, col, d32, areas


def test_colours_as_features_are_the_colour_oracle(serial):
    sc, us, ci, col, d32, areas = _frame()
    al = sc["alphas"]
    ref = orc.splat(H, W, us, ci, al, d32.copy(), col, areas.copy())
    f = np.asarray(col, np.float32)
    got = ofe.splat_features(H, W, us, ci, al, d32, areas, f)
    assert np.array_equal(got["features"], ref["image"])
    for k in ("contrib", "final_tau", "ranges", "gsid", "ambiguous"):
        assert np.array_equal(got[k], ref[k]), k
    dl = upstream_gradient(W, H, 3).astype(np.float32) * (3.0 * W * H)
    want = orc.splat_backward(H, W, us, ci, al, f, ref, dl, return_ambiguous=True)
    back = ofe.splat_backward_features(H, W, us, ci, al, got, f, dl, return_ambiguous=True)
    for a, b, name in zip(back[:3], want[:3], ("dus", "dcinv2ds", "dalphas")):
        assert np.array_equal(a, b), name
    assert np.array_equal(back[3], want[3].reshape(-1, 3))
    assert np.array_equal(back[4], want[4])


def test_depth_and_one_as_features_are_the_rgbd_planes():
    sc, us, ci, col, d32, areas = _frame(seed=5)
    al = sc["alphas"]
    g = orgbd.splat_rgbd(H, W, us, ci, al, d32.copy(), col, areas.copy())
    z = np.asarray(g["z"], np.float32).reshape(-1, 1)
    fz = ofe.splat_features(H, W, us, ci, al, d32, areas, z)["features"][0]
    f1 = ofe.splat_features(H, W, us, ci, al, d32, areas, np.ones((N, 1), np.float32))["features"][0]
    assert np.abs(fz - g["depth"]).max() <= 1e-12 * max(np.abs(g["depth"]).max(), 1.0)
    assert np.abs(f1 - g["alpha"]).max() <= 1e-12
    assert g["alpha"].max() > 0.5


def test_channel_split_is_linear():
    sc, us, ci, col, d32, areas = _frame(seed=7)
    al = sc["alphas"]
    rng = np.random.default_rng(1)
    f = rng.normal(size=(N, 7)).astype(np.float32)
    dF = rng.normal(size=(7, H, W)).astype(np.float32)
    one = ofe.splat_features(H, W, us, ci, al, d32, areas, f)
    a = ofe.splat_features(H, W, us, ci, al, d32, areas, f[:, :4])
    b = ofe.splat_features(H, W, us, ci, al, d32, areas, f[:, 4:])
    assert np.array_equal(np.concatenate([a["features"], b["features"]]), one["features"])
    g1 = ofe.splat_backward_features(H, W, us, ci, al, one, f, dF)
    ga = ofe.splat_backward_features(H, W, us, ci, al, one, f[:, :4], dF[:4])
    gb = ofe.splat_backward_features(H, W, us, ci, al, one, f[:, 4:], dF[4:])
    for x, y, z in zip(g1[:3], ga[:3], gb[:3]):
        assert np.abs(x - (y + z)).max() <= 1e-11 * max(np.abs(x).max(), 1e-30)
    assert np.abs(g1[3] - np.concatenate([ga[3], gb[3]], axis=1)).max() <= 1e-12 * np.abs(g1[3]).max()


def test_feature_gradients_vs_central_differences():
    """L = <G, F>: the oracle's dL/dus, dL/dconic, dL/dalpha and dL/dfeatures against central
    differences of its own forward, in the pattern of test_oracle_fd.py"""
    n, w, h, D = 120, 48, 40, 5
    sc, us, ci, col, d32, areas = _frame(seed=11, n=n, w=w, h=h)
    rng = np.random.default_rng(2)
    f = rng.normal(size=(n, D))
    G = rng.normal(size=(D, h, w))
    X = {"us": np.asarray(us, np.float64).copy(), "ci": np.asarray(ci, np.float64).copy(),
         "al": np.asarray(sc["alphas"], np.float64).reshape(-1).copy(), "f": f}

    def fwd():
        return ofe.splat_features(h, w, X["us"], X["ci"], X["al"], d32, areas, X["f"])

    def loss():
        return float((fwd()["features"] * G).sum())

    ref = fwd()
    du, dc, da, dfeat = ofe.splat_backward_features(h, w, X["us"], X["ci"], X["al"], ref, X["f"], G)
    grads = {"us": du.reshape(n, 2), "ci": dc.reshape(n, 3), "al": da.reshape(n), "f": dfeat}
    used = np.unique(ref["gsid"])
    L0 = loss()
    picks = [(("us", "ci", "al", "f")[rng.integers(4)], int(rng.choice(used))) for _ in range(64)]
    good = 0
    for name, i in picks:
        x = X[name]
        idx = (i,) if name == "al" else (i, int(rng.integers(x.shape[1])))
        x0 = float(x[idx])
        an = float(grads[name][idx])
        for rel in (2e-3, 5e-4, 1.5e-4):  # piecewise smooth, fp32-rounded inputs (test_oracle_fd.py)
            hstep = rel * max(abs(x0), 0.05)
            x[idx] = x0 + hstep
            lp = loss()
            x[idx] = x0 - hstep
            lm = loss()
            x[idx] = x0
            fd = (lp - lm) / (2 * hstep)
            if abs(fd - an) <= 1e-2 * max(abs(fd), abs(an)) + 1e-6 * abs(L0):
                good += 1
                break
    assert good >= int(0.85 * len(picks)), "only %d of %d finite differences agree" % (good, len(picks))


# ---------------------------------------------------------------- the C ABI and the sm_90a binary
def test_feature_symbols_signatures_and_workspace_queries():
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    lib = _lib.load()
    syms = header_symbols()
    for s in ("gsb_splat_features", "gsb_splat_features_backward", "gsb_splat_features_workspace_bytes",
              "gsb_density_apply_rows"):
        assert s in syms and s in _lib.SIGNATURES and hasattr(lib, s), s
    # host-only answers: the work area grows with the tile grid, the records with N when re-packed
    a = lib.gsb_splat_features_workspace_bytes(1000, 64, 64, 0)
    b = lib.gsb_splat_features_workspace_bytes(1000, 64, 64, 5000)
    c = lib.gsb_splat_features_workspace_bytes(1000, 1080, 1920, 0)
    assert a >= (4 * 16 + 2) * 4 and b >= 48 * 1000 + (4 * 16 + 2) * 4 and c >= (4 * 68 * 120 + 2) * 4
    # argument errors are found before any device work
    vp = C.c_void_p
    ws = (C.c_char * 4096)()
    rc = lib.gsb_splat_features(16, 16, 0, 0, 0, None, None, None, None, None, None, vp(16), vp(16), None,
                                C.cast(ws, vp), 4096, vp(256), None)
    assert rc != 0 and b"D < 1" in lib.gsb_last_error()
    rc = lib.gsb_splat_features(16, 16, 0, 0, 3, None, None, None, None, None, None, vp(16), vp(16), None,
                                C.cast(ws, vp), 4096, vp(260), None)
    assert rc != 0 and b"misaligned feature_image" in lib.gsb_last_error()
    rc = lib.gsb_splat_features(16, 16 * 65536, 0, 0, 3, None, None, None, None, None, None, vp(16), vp(16), None,
                                C.cast(ws, vp), 4096, vp(256), None)
    assert rc != 0 and b"65535 tiles" in lib.gsb_last_error()
    rc = lib.gsb_density_apply_rows(10, vp(16), vp(16), 5, 1, 1, 0, vp(16), None, None, vp(16), None, None, None)
    assert rc != 0 and b"bad counts" in lib.gsb_last_error()
    assert lib.gsb_density_apply_rows(0, None, None, 0, 0, 0, 4, None, None, None, None, None, None, None) == 0


def test_feature_rasterizers_are_sm90a_without_spills():
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    for name in ("k_draw_feat", "k_draw_feat_bwd"):
        for G in (4, 8):
            body = [f for f in funcs if f.startswith("_ZN3gsb%d%sILi%dEE" % (len(name), name, G))]
            assert len(body) == 1, (name, G)
            for op in ("LDGSTS.E.BYPASS.128", "LDGDEPBAR", "DEPBAR.LE", "MUFU.EX2"):
                assert op in body[0], "%s<%d>: %s missing" % (name, G, op)
    assert set(re.findall(r"code for (sm_\w+)", sass)) == {"sm_90a"}
    r = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True)
    found = re.findall(r"Function (_ZN3gsb\d+k_draw_feat\w*|\S*k_density_copy_rows\S*):\s*\n\s*(REG:.*)", r.stdout)
    assert len(found) == 5, found
    for name, usage in found:
        assert "LOCAL:0 " in usage and "STACK:0 " in usage, (name, usage)
    lib = _lib.load()
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    assert names.index("draw") == 11 and names.index("draw_backward") == 12
    assert "draw_features" in names and "draw_backward_features" in names and "density_apply_rows" in names
    assert names[-2:] == ["draw_rgbd", "draw_backward_rgbd"]
