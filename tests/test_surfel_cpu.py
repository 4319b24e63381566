"""2D Gaussian Splatting without a GPU: the fp64 oracle's analytic backward against central
differences of its own forward (every parameter, the screen-space shift, SH degrees 0-3, an
edge-on and a clamped surfel), and the C ABI of the surfel entry points."""
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import surfel_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, W = 20, 36  # not multiples of 16
FX = FY = 30.0
CX, CY = 17.3, 9.6


def scene(k, seed=0):
    rng = np.random.default_rng(seed)
    N = 6
    pws = np.stack([rng.uniform(-0.8, 0.8, N), rng.uniform(-0.4, 0.4, N), rng.uniform(2.5, 4.0, N)], 1)
    rots = rng.normal(size=(N, 4))
    # surfel 0 edge-on: its normal R e2 along x, the view along z
    rots[0] = [np.cos(np.pi / 4), 0.0, np.sin(np.pi / 4), 0.0]
    pws[0] = [0.1, 0.05, 3.0]
    scales = np.stack([rng.uniform(0.15, 0.4, N), rng.uniform(0.15, 0.4, N), rng.uniform(0.0, 0.1, N)], 1)
    shs = rng.normal(scale=0.4, size=(N, 3 * k))
    alphas = rng.uniform(0.3, 0.9, N)
    alphas[1] = 0.9985  # clamped near its centre
    Rcw = np.eye(3)
    tcw = np.zeros(3)
    twc = np.zeros(3)
    return dict(pws=pws, rots=rots, scales=scales, shs=shs, alphas=alphas, Rcw=Rcw, tcw=tcw, twc=twc)


def planes(seed):
    rng = np.random.default_rng(seed + 100)
    return (rng.normal(size=(3, H, W)), rng.normal(size=(H, W)), rng.normal(size=(H, W)), rng.normal(size=(3, H, W)))


def loss(sc, bins, dl, delta=None):
    pre = so.preprocess(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], FX, FY, CX, CY)
    out = so.render(H, W, pre, sc["alphas"], bins, delta=delta)
    return (np.sum(out["image"] * dl[0]) + np.sum(out["depth"] * dl[1]) + np.sum(out["alpha"] * dl[2]) +
            np.sum(out["normal"] * dl[3])), out


@pytest.mark.parametrize("k", [1, 4, 9, 16])
def test_oracle_backward_matches_central_differences(k):
    sc = scene(k, seed=k)
    dl = planes(k)
    pre = so.preprocess(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], FX, FY, CX, CY)
    assert pre["keep"].all()
    bins = so.bin_f32(H, W, pre)
    assert bins[0] > 0
    fwd = so.render(H, W, pre, sc["alphas"], bins)
    assert not fwd["ambiguous"].any()
    assert (fwd["alpha"] > 0).mean() > 0.3
    rows = so.render_backward(H, W, pre, sc["alphas"], bins, fwd, *dl)
    g = so.preprocess_backward(pre, rows)
    # the edge-on surfel is drawn through its screen-space filter; the clamped one reaches 0.99
    e0 = so._eval(pre["M"][0], pre["u"][0], pre["u"][0][0] + np.array([1.5, -2.0]), pre["u"][0][1] + np.array([0.7, 1.0]))
    assert not e0["b3"].any()
    assert (np.asarray(sc["alphas"][1]) * np.exp(-0.5 * so._eval(pre["M"][1], pre["u"][1], pre["u"][1][:1],
                                                                  pre["u"][1][1:])["G"]) > so.ALPHA_CLAMP).all()
    eps = 1e-6
    checks = [("pws", sc["pws"], None), ("shs", sc["shs"], None), ("alphas", sc["alphas"], None),
              ("scales", sc["scales"], [0, 1]), ("rots", sc["rots"], None)]
    for name, arr, cols in checks:
        fd = np.zeros_like(arr)
        it = np.ndindex(arr.shape)
        for idx in it:
            if cols is not None and idx[1] not in cols:
                continue
            keep = arr[idx]
            arr[idx] = keep + eps
            lp, _ = loss(sc, bins, dl)
            arr[idx] = keep - eps
            lm, _ = loss(sc, bins, dl)
            arr[idx] = keep
            fd[idx] = (lp - lm) / (2 * eps)
        an = g[name].reshape(arr.shape)
        if cols is not None:
            an = an[:, cols]
            fd = fd[:, cols]
        scale = np.abs(fd).max()
        assert scale > 0, name
        np.testing.assert_allclose(an, fd, atol=2e-5 * scale + 1e-7, err_msg=name)
    # dL/ddelta: the whole surfel shifted in screen space
    fd = np.zeros((len(sc["alphas"]), 2))
    for i in range(fd.shape[0]):
        for c in range(2):
            d = np.zeros_like(fd)
            d[i, c] = eps
            lp, _ = loss(sc, bins, dl, d)
            lm, _ = loss(sc, bins, dl, -d)
            fd[i, c] = (lp - lm) / (2 * eps)
    np.testing.assert_allclose(g["us"], fd, atol=2e-5 * np.abs(fd).max(), err_msg="delta")


def test_fronto_parallel_identities():
    """surfels parallel to the image plane at one depth z0: depth = z0 alpha, normal = (0, 0, -alpha)"""
    rng = np.random.default_rng(3)
    N, z0 = 8, 3.0
    pws = np.stack([rng.uniform(-0.6, 0.6, N), rng.uniform(-0.3, 0.3, N), np.full(N, z0)], 1)
    ang = rng.uniform(0, np.pi, N)
    rots = np.stack([np.cos(ang / 2), np.zeros(N), np.zeros(N), np.sin(ang / 2)], 1)  # about the view axis
    scales = np.stack([rng.uniform(0.1, 0.3, N), rng.uniform(0.1, 0.3, N), np.zeros(N)], 1)
    pre = so.preprocess(pws, rots, scales, rng.normal(size=(N, 3)), np.eye(3), np.zeros(3), np.zeros(3), FX, FY, CX, CY)
    bins = so.bin_f32(H, W, pre)
    out = so.render(H, W, pre, rng.uniform(0.2, 0.9, N), bins)
    np.testing.assert_allclose(out["depth"], z0 * out["alpha"], atol=1e-12)
    np.testing.assert_allclose(out["normal"][2], -out["alpha"], atol=1e-12)
    np.testing.assert_allclose(out["normal"][:2], 0, atol=1e-12)


def _header_decls():
    src = open(os.path.join(ROOT, "include", "gsplat_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return {m.group(1): m.group(2) for m in re.finditer(r"\b(gsb_[a-z0-9_]*surfel[a-z0-9_]*)\s*\(([^;]*)\)\s*;", src)}


def test_surfel_abi_symbols_signatures_and_workspace():
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    lib = _lib.load()
    decls = _header_decls()
    assert sorted(decls) == sorted(["gsb_surfel_preprocess_forward", "gsb_surfel_preprocess_backward",
                                    "gsb_splat_surfel_workspace_bytes", "gsb_splat_surfel_render",
                                    "gsb_splat_surfel_forward", "gsb_splat_surfel_backward"])
    for name, args in decls.items():
        assert name in _lib.SIGNATURES
        assert len(_lib.SIGNATURES[name][1]) == len(args.split(",")), name
    assert lib.gsb_abi_version() == 1
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    assert names.index("draw") == 11
    for n in ("surfel_forward", "draw_surfel", "draw_surfel_backward", "surfel_backward"):
        assert names.index(n) < names.index("draw_backward_abs")
    small = lib.gsb_splat_surfel_workspace_bytes(1000, 64, 64, 0)
    assert small >= (2 + 4 * 16) * 4
    assert lib.gsb_splat_surfel_workspace_bytes(1000, 64, 64, 100000) > small
    # argument errors answer without a GPU
    assert lib.gsb_splat_surfel_render(0, 64, 10, 0, 0, *([None] * 5), 0, *([None] * 9)) == -1
    assert b"bad N/H/W" in lib.gsb_last_error()
    assert lib.gsb_splat_surfel_backward(64, 64, -1, 0, *([None] * 10), 0, None, None) == -1
    assert lib.gsb_surfel_preprocess_forward(4, 2, *([None] * 7), *([1.0] * 6), *([None] * 7)) == -1
    assert b"1, 4, 9 or 16" in lib.gsb_last_error()


def test_surfel_kernels_sass():
    """both rasterizers gather with cp.async (LDGSTS + LDGDEPBAR / DEPBAR) and use MUFU.EX2; every
    surfel kernel is sm_90a code without local memory"""
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    r = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True)
    assert r.returncode == 0
    funcs = {}
    cur = None
    for ln in r.stdout.splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur is not None:
            funcs[cur].append(ln)
    for kname in ("k_draw_surfelE", "k_draw_surfel_bwdE"):
        body = [b for f, b in funcs.items() if kname in f]
        assert len(body) == 1, kname
        text = "\n".join(body[0])
        for ins in ("LDGSTS.E.BYPASS.128", "LDGDEPBAR", "DEPBAR.LE", "MUFU.EX2"):
            assert ins in text, (kname, ins)
    arch = subprocess.run(["cuobjdump", "-lelf", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in arch and not re.search(r"sm_(?!90a)\d+", arch)
    res = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True).stdout
    lines = res.splitlines()
    seen = 0
    for i, ln in enumerate(lines):
        if "Function" in ln and "surfel" in ln:
            seen += 1
            assert "LOCAL:0" in lines[i + 1] and "STACK:0" in lines[i + 1], ln
    assert seen == 10
