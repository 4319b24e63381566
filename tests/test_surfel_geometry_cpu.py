"""2DGS geometry terms (DESIGN 3.16) without a GPU: the fp64 model (tests/surfel_geometry_oracle.py)
against brute force and against central differences of itself, loss.depth_to_normal on analytic
planes, and the C ABI of gsb_splat_2dgs_* (symbols, argument errors, profile ids, SASS)."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import surfel_oracle as so
import surfel_geometry_oracle as sg
from test_surfel_edge_scenes_cpu import (CX, CY, FX, FY, H, W, camera, fd_scene, fronto, place, quat, random_scene,
                                         rot)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------- the model against brute force
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_geometry_matches_brute_force(seed):
    """per pixel, the contributing records found by a plain walk (their w, m, z and incoming tau):
    the O(K^2) double sum and the median found by scanning tau agree with render_geometry"""
    sc = random_scene(60, 40, 28, 1, cam="posed_a", seed=seed, z=(1.0, 4.0), alpha=(0.2, 0.99))
    pre = so.preprocess(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                        sc["fy"], sc["cx"], sc["cy"])
    bins = so.bin_f32(28, 40, pre)
    near, far = 1.5, 20.0
    out = sg.render_geometry(28, 40, pre, sc["alphas"], bins, near, far)
    _, ranges, gsid, _ = bins
    gx = (40 + 15) // 16
    checked = 0
    for y in range(28):
        for x in range(40):
            t = (y // 16) * gx + x // 16
            tau, ws, ms, zs, taus, idxs = 1.0, [], [], [], [], []
            for j, i in enumerate(gsid[ranges[t, 0]:ranges[t, 1]]):
                e = so._eval(pre["M"][i], pre["u"][i], np.array([float(x)]), np.array([float(y)]))
                ap = min(so.ALPHA_CLAMP, float(sc["alphas"][i]) * np.exp(-0.5 * e["G"][0]))
                if tau < so.TAU_STOP or ap < so.ALPHA_SKIP:
                    continue
                z = e["z"][0]
                ws.append(tau * ap); ms.append(far / (far - near) * (1 - near / max(z, near))); zs.append(z)
                taus.append(tau); idxs.append(j)
                tau *= 1 - ap
            dist, med, medc = sg.brute_force(ws, ms, zs, taus, idxs)
            assert abs(out["distortion"][y, x] - dist) <= 1e-12 * max(1.0, dist), (x, y)
            assert out["median_depth"][y, x] == med and out["median_contrib"][y, x] == medc, (x, y)
            assert abs(out["moments"][0, y, x] - sum(w * m for w, m in zip(ws, ms))) < 1e-12
            checked += len(ws) > 1
    assert checked > 200
    assert (out["distortion"] > 0).mean() > 0.3 and (out["median_contrib"] > 0).mean() > 0.5
    # the surfel planes are surfel_oracle's
    ref = so.render(28, 40, pre, sc["alphas"], bins)
    for k in ("image", "depth", "alpha", "normal", "contrib", "final_tau"):
        np.testing.assert_array_equal(out[k], ref[k])


# ---------------------------------------------------------------- the model's backward
NEAR, FAR = 2.9, 50.0


def geo_scene(k, cam, seed):
    """fd_scene (edge-on, clamped, flipped surfels) + a stack of three near-opaque fronto-parallel
    disks at z 2.2-2.3 whose centre pixels stop on tau, all at NEAR = 2.9: hits on both sides of near"""
    sc = fd_scene(k, cam, seed)
    Rcw, tcw, _ = camera(cam)
    pc = np.array([[0.25, -0.12, 2.2], [0.25, -0.12, 2.25], [0.25, -0.12, 2.3]])
    rng = np.random.default_rng(seed + 99)
    sc["pws"] = np.concatenate([sc["pws"], (pc - tcw) @ Rcw])
    sc["rots"] = np.concatenate([sc["rots"], np.stack([quat(Rcw.T @ rot([0.2, 0.1, 0.3], 0.1 * j) @ fronto(1)[0])
                                                       for j in range(3)])])
    sc["scales"] = np.concatenate([sc["scales"], [[0.25, 0.22, 0.0], [0.24, 0.26, 0.0], [0.27, 0.23, 0.0]]])
    sc["shs"] = np.concatenate([sc["shs"], rng.normal(scale=0.4, size=(3, 3 * k))])
    sc["alphas"] = np.concatenate([sc["alphas"], [0.97, 0.96, 0.975]])
    return sc


def geo_loss(sc, bins, dl, delta=None):
    pre = so.preprocess(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], FX, FY, CX, CY)
    out = sg.render_geometry(H, W, pre, sc["alphas"], bins, NEAR, FAR, delta=delta)
    return (np.sum(out["image"] * dl[0]) + np.sum(out["depth"] * dl[1]) + np.sum(out["alpha"] * dl[2]) +
            np.sum(out["normal"] * dl[3]) + np.sum(out["distortion"] * dl[4]) + np.sum(out["median_depth"] * dl[5]))


@pytest.mark.parametrize("planes", ["distortion", "median", "all"])
@pytest.mark.parametrize("k", [1, 4, 9, 16])
def test_oracle_geometry_backward_matches_central_differences(k, planes):
    sc = geo_scene(k, "posed_a", seed=3 * k + 1)
    rng = np.random.default_rng(k + 70)
    full = [rng.normal(size=(3, H, W)), rng.normal(size=(H, W)), rng.normal(size=(H, W)), rng.normal(size=(3, H, W)),
            rng.normal(size=(H, W)) * 20.0, rng.normal(size=(H, W))]
    use = {"distortion": (4,), "median": (5,), "all": range(6)}[planes]
    dl = [a if i in use else np.zeros_like(a) for i, a in enumerate(full)]
    pre = so.preprocess(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], FX, FY, CX, CY)
    assert pre["keep"].all()
    bins = so.bin_f32(H, W, pre)
    fwd = sg.render_geometry(H, W, pre, sc["alphas"], bins, NEAR, FAR)
    assert not fwd["ambiguous"].any()
    # the scene's edges: a pixel that stops on tau before its list ends, hits below near, the clamp
    lens = np.diff(bins[1], axis=1)[:, 0]
    tile = lambda y, x: (y // 16) * ((W + 15) // 16) + x // 16
    stops = [(y, x) for y in range(H) for x in range(W)
             if fwd["final_tau"][y, x] < so.TAU_STOP and fwd["contrib"][y, x] < lens[tile(y, x)]]
    assert stops
    below = 0
    for i in range(len(sc["alphas"])):
        ys, xs = np.mgrid[0:H, 0:W]
        e = so._eval(pre["M"][i], pre["u"][i], xs.ravel().astype(float), ys.ravel().astype(float))
        below += np.sum((e["z"] < NEAR) & (sc["alphas"][i] * np.exp(-0.5 * e["G"]) > 0.01))
    assert below > 0 and (fwd["distortion"] > 0).mean() > 0.2
    rows = sg.render_backward_geometry(H, W, pre, sc["alphas"], bins, fwd, *dl, near=NEAR, far=FAR)
    g = so.preprocess_backward(pre, rows)
    eps = 1e-6
    for name, cols in (("pws", None), ("shs", None), ("alphas", None), ("scales", [0, 1]), ("rots", None)):
        arr = sc[name]
        fd = np.zeros_like(arr)
        for idx in np.ndindex(arr.shape):
            if cols is not None and idx[1] not in cols:
                continue
            keep = arr[idx]
            arr[idx] = keep + eps
            lp = geo_loss(sc, bins, dl)
            arr[idx] = keep - eps
            lm = geo_loss(sc, bins, dl)
            arr[idx] = keep
            fd[idx] = (lp - lm) / (2 * eps)
        an = g[name].reshape(arr.shape)
        if cols is not None:
            an, fd = an[:, cols], fd[:, cols]
        # the geometry planes do not see colour, and the median is piecewise constant in alpha
        if (name == "shs" and planes != "all") or (name == "alphas" and planes == "median"):
            assert not an.any() and not fd.any()
            continue
        scale = np.abs(fd).max()
        assert scale > 0, name
        np.testing.assert_allclose(an, fd, atol=2e-5 * scale + 1e-7, err_msg=name)
    N = len(sc["alphas"])
    fd = np.zeros((N, 2))
    for i in range(N):
        for c_ in range(2):
            d = np.zeros((N, 2))
            d[i, c_] = eps
            fd[i, c_] = (geo_loss(sc, bins, dl, d) - geo_loss(sc, bins, dl, -d)) / (2 * eps)
    np.testing.assert_allclose(g["us"], fd, atol=2e-5 * np.abs(fd).max(), err_msg="delta")


@pytest.mark.parametrize("k,cam,seed", [(1, "posed_a", 2), (4, "posed_b", 5), (9, "posed_a", 8), (16, "posed_b", 11)])
def test_oracle_geometry_backward_without_geometry_is_surfel_oracles(k, cam, seed):
    """render_backward_geometry restates surfel_oracle.render_backward with the geometry terms added:
    without them it must give the same rows, on every scene the geometry tests use"""
    sc = geo_scene(k, cam, seed=seed)
    rng = np.random.default_rng(seed)
    dl = [rng.normal(size=(3, H, W)), rng.normal(size=(H, W)), rng.normal(size=(H, W)), rng.normal(size=(3, H, W))]
    pre = so.preprocess(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], FX, FY, CX, CY)
    bins = so.bin_f32(H, W, pre)
    fwd = sg.render_geometry(H, W, pre, sc["alphas"], bins, NEAR, FAR)
    ref, ref_abs = so.render_backward(H, W, pre, sc["alphas"], bins, fwd, *dl, abs_rows=True)
    got, got_abs = sg.render_backward_geometry(H, W, pre, sc["alphas"], bins, fwd, *dl, near=NEAR, far=FAR,
                                               abs_rows=True)
    np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-12 * np.abs(ref).max())
    assert (got_abs >= ref_abs * (1 - 1e-12)).all()
    got, got_abs = sg.render_backward_geometry(H, W, pre, sc["alphas"], bins, fwd, *dl, rng.normal(size=(H, W)),
                                               rng.normal(size=(H, W)), near=NEAR, far=FAR, abs_rows=True)
    assert (got_abs >= np.abs(got) * (1 - 1e-12)).all()


# ---------------------------------------------------------------- depth_to_normal
class _Cam:
    width, height, fx, fy, cx, cy = 48, 36, 40.0, 44.0, 23.4, 17.7


def _plane_depth(n, d, cam, dtype=torch.float64):
    """depth of the plane n . X = d along each pixel's ray (X = z K^-1 (u, v, 1))"""
    v, u = torch.meshgrid(torch.arange(cam.height, dtype=dtype), torch.arange(cam.width, dtype=dtype), indexing="ij")
    r = torch.stack([(u - cam.cx) / cam.fx, (v - cam.cy) / cam.fy, torch.ones_like(u)])
    return d / (n[0] * r[0] + n[1] * r[1] + n[2] * r[2])


@pytest.mark.parametrize("n", [(0.0, 0.0, -1.0), (0.3, -0.2, -0.93), (-0.45, 0.1, 0.88), (0.05, 0.6, -0.8)])
def test_depth_to_normal_on_analytic_planes(n):
    from easygaussiansplatting_b200.loss import depth_to_normal
    cam = _Cam()
    nv = torch.tensor(n, dtype=torch.float64)
    nv = nv / nv.norm()
    d = -3.0 if nv[2] < 0 else 3.0   # the plane in front of the camera
    depth = _plane_depth(nv, d, cam)
    assert (depth > 0).all()
    got = depth_to_normal(depth, cam)
    assert got.shape == (3, cam.height, cam.width)
    want = nv if nv[2] < 0 else -nv   # facing the camera
    inner = got[:, 1:-1, 1:-1]
    assert torch.allclose(inner, want[:, None, None].expand_as(inner), atol=1e-9)
    for border in (got[:, 0], got[:, -1], got[:, :, 0], got[:, :, -1]):
        assert (border == 0).all()
    if n == (0.0, 0.0, -1.0):
        assert torch.equal(got[:, 1:-1, 1:-1].round(decimals=12),
                           torch.tensor([0.0, 0.0, -1.0], dtype=torch.float64)[:, None, None].expand_as(inner))


def test_depth_to_normal_degenerate_pixels_have_bounded_gradients():
    """a one-pixel covered row over empty pixels (depth 0), holes, and a covered column: the pixels
    without a surface around them get a zero normal and no gradient; 2DGS's normal term stays bounded"""
    from easygaussiansplatting_b200.loss import depth_to_normal

    class Cam:
        width, height, fx, fy, cx, cy = 8, 7, 6.0, 6.5, 3.7, 3.2

    rng = np.random.default_rng(4)
    row = np.zeros((7, 8))
    row[3] = 2.0 + rng.uniform(0, 0.3, 8)
    col = np.zeros((7, 8))
    col[:, 4] = 2.0 + rng.uniform(0, 0.3, 7)
    holes = 2.0 + rng.uniform(0, 0.3, (7, 8))
    holes[2, 3] = holes[4, 5] = holes[5, 1] = 0.0
    for d0 in (row, col, holes):
        depth = torch.tensor(d0, dtype=torch.float64, requires_grad=True)
        normal = torch.tensor(rng.normal(size=(3, 7, 8)), dtype=torch.float64)
        alpha = torch.tensor(rng.uniform(0.2, 1.0, (7, 8)), dtype=torch.float64)
        nd = depth_to_normal(depth, Cam())
        loss = (1 - (normal * nd * alpha.detach()).sum(0)).mean()
        (g,) = torch.autograd.grad(loss, depth)
        assert torch.isfinite(nd).all() and torch.isfinite(g).all()
        assert g.abs().max() < 10.0, float(g.abs().max())
        inner = nd[:, 1:-1, 1:-1]
        d = depth.detach()
        bad = ((d[1:-1, 1:-1] <= 0) | (d[1:-1, 2:] <= 0) | (d[1:-1, :-2] <= 0) | (d[2:, 1:-1] <= 0) |
               (d[:-2, 1:-1] <= 0))
        assert (inner[:, bad] == 0).all()
        n_ok = inner[:, ~bad]
        assert torch.allclose(n_ok.norm(dim=0), torch.ones(n_ok.shape[1], dtype=torch.float64))
        if d0 is holes:
            assert (~bad).sum() > 5
        else:   # every interior pixel of a one-pixel strip lacks a neighbour: no gradient at all
            assert bad.all() and not g.any()


def test_depth_to_normal_gradcheck():
    from easygaussiansplatting_b200.loss import depth_to_normal

    class Cam:
        width, height, fx, fy, cx, cy = 7, 6, 5.0, 6.0, 3.2, 2.9

    rng = np.random.default_rng(0)
    depth = torch.tensor(2.0 + rng.uniform(0, 0.5, (6, 7)), dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(lambda d: depth_to_normal(d, Cam()), (depth,))


# ---------------------------------------------------------------- the C ABI
NEW = ("gsb_splat_2dgs_render", "gsb_splat_2dgs_forward", "gsb_splat_2dgs_backward")


def _decls():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "gsplat_b200.h")).read(), flags=re.S)
    return {m.group(1): m.group(2) for m in re.finditer(r"\b(gsb_splat_2dgs_\w+)\s*\(([^;]*)\)\s*;", src)}


def test_2dgs_abi_symbols_and_profile_ids():
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    lib = _lib.load()
    decls = _decls()
    assert sorted(decls) == sorted(NEW)
    syms = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    for name, args in decls.items():
        assert len(_lib.SIGNATURES[name][1]) == len(args.split(",")), name
        assert re.search(r"\bT %s$" % name, syms, re.M), name
        assert "surfel" not in name
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    i = names.index("surfel_backward")
    assert names[i + 1:i + 4] == ["draw_2dgs", "draw_2dgs_backward", "draw_backward_abs"]


PTR = 0x10000000
MIS16 = PTR + 8
MIS4 = PTR + 2   # not even float-aligned
BIG = 1 << 40
NAN, INF = float("nan"), float("inf")

CASES = [
    ("gsb_splat_2dgs_render", {"H": 0}, "splat: bad N/H/W"),
    ("gsb_splat_2dgs_render", {"P": -1}, "splat_2dgs: bad P"),
    ("gsb_splat_2dgs_render", {"records": None}, "splat_2dgs: null pointer"),
    ("gsb_splat_2dgs_render", {"near": 0.0}, "splat_2dgs: near <= 0"),
    ("gsb_splat_2dgs_render", {"near": -1.0}, "splat_2dgs: near <= 0"),
    ("gsb_splat_2dgs_render", {"far": 0.1}, "splat_2dgs: far <= near"),
    ("gsb_splat_2dgs_render", {"far": 0.2}, "splat_2dgs: far <= near"),
    ("gsb_splat_2dgs_render", {"near": NAN}, "splat_2dgs: near / far not finite"),
    ("gsb_splat_2dgs_render", {"far": INF}, "splat_2dgs: near / far not finite"),
    ("gsb_splat_2dgs_render", {"distortion": None}, "splat_2dgs: null geometry plane"),
    ("gsb_splat_2dgs_render", {"median_contrib": None}, "splat_2dgs: null geometry plane"),
    ("gsb_splat_2dgs_render", {"moments": MIS16}, "splat_2dgs: misaligned geometry plane"),
    ("gsb_splat_2dgs_render", {"median_depth": MIS16}, "splat_2dgs: misaligned geometry plane"),
    ("gsb_splat_2dgs_render", {"image": None}, "splat_2dgs: null output"),
    ("gsb_splat_2dgs_render", {"normal_image": None}, "splat_2dgs: null output"),
    ("gsb_splat_2dgs_render", {"alpha_image": MIS16}, "splat_2dgs: misaligned output"),
    ("gsb_splat_2dgs_render", {"records": MIS16}, "splat_2dgs: records misaligned"),
    ("gsb_splat_2dgs_render", {"ws": MIS16}, "splat_2dgs: ws misaligned"),
    ("gsb_splat_2dgs_render", {"ws_bytes": 64}, "splat_2dgs: workspace too small"),
    ("gsb_splat_2dgs_forward", {"N": -1}, "splat: bad N/H/W"),
    ("gsb_splat_2dgs_forward", {"P_cap": 0}, "splat_2dgs_forward: bad P_cap"),
    ("gsb_splat_2dgs_forward", {"status_host": None}, "splat_2dgs_forward: null pointer"),
    ("gsb_splat_2dgs_forward", {"records": None}, "splat_2dgs_forward: null pointer"),
    ("gsb_splat_2dgs_forward", {"far": -INF}, "splat_2dgs: near / far not finite"),
    ("gsb_splat_2dgs_forward", {"near": 5.0, "far": 4.0}, "splat_2dgs: far <= near"),
    ("gsb_splat_2dgs_forward", {"moments": None}, "splat_2dgs: null geometry plane"),
    ("gsb_splat_2dgs_forward", {"distortion": MIS16}, "splat_2dgs: misaligned geometry plane"),
    ("gsb_splat_2dgs_backward", {"P": -1}, "splatB_2dgs: bad N/H/W/P"),
    ("gsb_splat_2dgs_backward", {"W": 16 * 65536}, "splatB_2dgs: more than 65535 tiles in a row or column"),
    ("gsb_splat_2dgs_backward", {"near": 0.0}, "splatB_2dgs: near <= 0"),
    ("gsb_splat_2dgs_backward", {"far": NAN}, "splatB_2dgs: near / far not finite"),
    ("gsb_splat_2dgs_backward", {"far": 0.1}, "splatB_2dgs: far <= near"),
    ("gsb_splat_2dgs_backward", {"rows": None}, "splatB_2dgs: null output"),
    ("gsb_splat_2dgs_backward", {"ws_bytes": 64}, "splatB_2dgs: workspace too small"),
    ("gsb_splat_2dgs_backward", {"gsid_per_patch": None}, "splatB_2dgs: null pointer"),
    ("gsb_splat_2dgs_backward", {"records": MIS16}, "splatB_2dgs: misaligned input"),
    ("gsb_splat_2dgs_backward", {"moments": None}, "splatB_2dgs: null geometry plane"),
    ("gsb_splat_2dgs_backward", {"median_contrib": None, "dloss_ddistortion": None},
     "splatB_2dgs: null geometry plane"),
    ("gsb_splat_2dgs_backward", {"alpha_image": MIS4}, "splatB_2dgs: misaligned geometry plane"),
    ("gsb_splat_2dgs_backward", {"moments": MIS4}, "splatB_2dgs: misaligned geometry plane"),
    ("gsb_splat_2dgs_backward", {"median_contrib": MIS4}, "splatB_2dgs: misaligned geometry plane"),
    ("gsb_splat_2dgs_backward", {"dloss_ddistortion": MIS4}, "splatB_2dgs: misaligned geometry plane"),
    ("gsb_splat_2dgs_backward", {"dloss_dmedian": MIS4, "dloss_ddistortion": None},
     "splatB_2dgs: misaligned geometry plane"),
]


def _param_names():
    return {k: [re.findall(r"\w+", p)[-1] for p in v.split(",")] for k, v in _decls().items()}


def _run_cases():
    import ctypes as C
    from easygaussiansplatting_b200 import _lib
    lib = _lib.load()
    names = _param_names()
    status = (C.c_uint32 * 4)()
    base = {"H": 64, "W": 64, "N": 10, "P": 100, "P_cap": 1000, "depth_key_max": 255, "depth_key_cap": 255,
            "ws_bytes": BIG, "bin_ws_bytes": BIG, "status_host": C.addressof(status), "stream": None,
            "near": 0.2, "far": 100.0}
    out = []
    for entry, broken, _ in CASES:
        args = {n: base.get(n, PTR) for n in names[entry]}
        assert set(broken) <= set(args), (entry, broken)
        args.update(broken)
        rc = getattr(lib, entry)(*args.values())
        out.append((rc, lib.gsb_last_error().decode()))
    return out


def test_2dgs_entry_points_name_the_failed_check():
    """every argument error answers -1 with its own text, in a process that sees no CUDA device"""
    from easygaussiansplatting_b200 import build
    build.build()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    r = subprocess.run([sys.executable, os.path.abspath(__file__)], capture_output=True, text=True, env=env, cwd=ROOT,
                       timeout=300)
    assert r.returncode == 0, r.stderr[-4000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    bad = [(e, b, want, tuple(g)) for (e, b, want), g in zip(CASES, got) if tuple(g) != (-1, "argument error: " + want)]
    assert len(got) == len(CASES) and not bad, "\n".join(map(str, bad))


def test_2dgs_kernels_sass():
    """both geometry rasterizers: sm_90a, cp.async gathers, MUFU.EX2, no local memory or stack;
    no new kernel carries 'surfel' in its name"""
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    funcs, cur = {}, None
    for ln in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur is not None:
            funcs[cur].append(ln)
    res = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True).stdout.splitlines()
    for kname in ("k_draw_2dgsE", "k_draw_2dgs_bwdE"):
        hits = [f for f in funcs if kname in f]
        assert len(hits) == 1, kname
        assert "surfel" not in hits[0]
        text = "\n".join(funcs[hits[0]])
        for ins in ("LDGSTS.E.BYPASS.128", "LDGDEPBAR", "DEPBAR.LE", "MUFU.EX2"):
            assert ins in text, (kname, ins)
        i = next(j for j, ln in enumerate(res) if "Function" in ln and hits[0] in ln)
        assert "LOCAL:0" in res[i + 1] and "STACK:0" in res[i + 1], res[i + 1]
    arch = subprocess.run(["cuobjdump", "-lelf", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in arch and not re.search(r"sm_(?!90a)\d+", arch)


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    print(json.dumps(_run_cases()))
