"""The 2DGS geometry terms (k_draw_2dgs, k_draw_2dgs_bwd, splat_surfel_geometry,
splatB_surfel_geometry, GSFunctionSurfelGeometry; DESIGN 3.16) at the surfel path's edges, against
the fp64 model of tests/surfel_geometry_oracle.py binned independently (so.bin_f32).  Scenes and
their model-only claims: tests/test_surfel_geometry_edge_scenes_cpu.py and
tests/test_surfel_edge_scenes_cpu.py.

1. Edge scenes through both geometry kernels at a (near, far) that cuts through the hits and one
   whose far lies below the farthest hits: the per-surfel outputs, the planes against the model per
   pixel, the rows per entry with all six upstream planes, and k_surfel_bwd on those rows per surfel;
   the hits at, below and beyond near / far, and near = 1e-3, far = 1e4; the last-column pixel pair.
2. Median ties, exactly: the strict tau > 0.5 at a tau of exactly 0.5, and dL/dmedian at one pixel
   reaching the median record's row alone.
3. Dead tiles at 4K and 1 km: every geometry plane, row and gradient of a dead surfel exactly 0.
4. Geometry planes over poisoned allocator memory: exactly 0 on tiles without patches.
5. The capacity path's rows against the exact path's, with both geometry gradients.
6. GSFunctionSurfelGeometry through autograd: the views autograd hands it, near / far reaching the
   backward, and 2DGS's training loss against the ops chain and the model."""
import numpy as np
import pytest
import torch

from oracle import surfel_oracle as so
import surfel_geometry_oracle as sg
from test_gpu_rgbd_edges import poison
from test_gpu_surfel_edges import (T, cam_args, check_preprocess, gpu_preprocess, n, ops, params, pre_of, record_pre,
                                   rows_bound, tile_map)
from test_gpu_surfel_geometry import check_geometry, check_rows, geo_frame
from test_surfel_edge_scenes_cpu import DEAD_H, DEAD_W, dead_claims, dead_scene, random_scene
from test_surfel_geometry_edge_scenes_cpu import (EDGE_SCENES, EXTREME, NF_FAR, NF_NEAR, TIE_LEN, coplanar_scene,
                                                  edge_scene, extreme_scene, near_far_pairs, near_far_scene, tie_claims,
                                                  tie_stacks)

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def upstream6(H, W, seed, ok=None):
    """random upstream planes for image, depth, alpha, normal, distortion (x10) and median, zero off ok"""
    rng = np.random.default_rng(seed)
    full = [rng.normal(size=(3, H, W)), rng.normal(size=(H, W)), rng.normal(size=(H, W)), rng.normal(size=(3, H, W)),
            rng.normal(size=(H, W)) * 10, rng.normal(size=(H, W))]
    return full if ok is None else [np.where(ok, a, 0.0) for a in full]


def bwd_args(res):
    """splatB_surfel_geometry's forward arguments from a geo_frame: records, contrib, final_tau, ranges,
    gsid, alpha, moments, median_contrib"""
    g, out = res
    return (g[4], out[1], out[2], out[3], out[4], out[6], out[10], out[11])


# ---------------------------------------------------------------- 1. edge scenes
@pytest.mark.parametrize("pair", [0, 1])
@pytest.mark.parametrize("name", EDGE_SCENES)
def test_edge_scenes_through_both_geometry_kernels(name, pair):
    """at both (near, far) pairs of near_far_pairs (hits on both sides of near; hits beyond far: shown on
    the model by test_geometry_claims_on_the_edge_scenes)"""
    sc = edge_scene(name)
    near, far = near_far_pairs(sc)[pair]
    check_preprocess(sc)
    res = check_geometry(sc, near, far)
    check_rows(sc, res, upstream6(sc["H"], sc["W"], len(sc["pws"]) + pair, res["ok"]), near, far)


@pytest.mark.parametrize("name", ["near_far", "extreme", "coplanar"])
def test_hits_at_below_and_beyond_near_and_far(name):
    """hits exactly at near (m and dm 0 on both sides), tiles whose every hit lies below near, hits beyond
    far; near = 1e-3, far = 1e4 (every m within 1e-3 of 1: the moment form cancels, held to the pixel's
    conditioning by check_geometry); coplanar disks (distortion 0 up to that bound)"""
    if name == "near_far":
        sc, (near, far) = near_far_scene(), (NF_NEAR, NF_FAR)
    elif name == "extreme":
        sc, (near, far) = extreme_scene(), EXTREME
    else:
        sc, (near, far) = coplanar_scene()[0], (0.2, 100.0)
    res = check_geometry(sc, near, far)
    H, W = sc["H"], sc["W"]
    if name == "near_far":
        # the pixels with a hit exactly at near, compared too: the model reports them instead of flagging
        fx = sg.render_geometry(H, W, res["rp"], sc["alphas"], res["bins"], near, far, exact=True)
        at = fx["at_near"] & ~fx["ambiguous"]
        assert at.sum() > 30
        dist, med, mom, medc = (n(x) for x in res["out"][8:])
        A, D, D2 = fx["alpha"], fx["moments"][0], fx["moments"][1]
        tol = 1e-4 * 2 * (A * D2 + D * D) + 2.0 ** -20 * A * A + 1e-30
        assert (np.abs(dist - fx["distortion"]) <= tol)[at].all()
        for k in range(2):
            assert (np.abs(mom[k] - fx["moments"][k]) <= 1e-4 * fx["moments"][k] + 2.0 ** -20 * A + 1e-30)[at].all()
        assert (medc == fx["median_contrib"])[at].all()
        below = (fx["contrib"] > 0) & (np.arange(W)[None, :] // 16 == 1)
        assert below.sum() > 30 and not dist[below].any() and not mom[:, below].any() and (med[below] > 0).all()
        ok = ~fx["ambiguous"]
        res["ok"] = ok
    check_rows(sc, res, upstream6(H, W, 40 + len(name), res["ok"]), near, far)


def test_backward_takes_up_no_pixel_past_the_last_column():
    """an odd frame width: the last column's pixel pair has no second pixel (bp.in1 false), and
    k_draw_2dgs_bwd must take up nothing of it.  Every plane the backward reads per pixel (contrib,
    final_tau, the six upstream planes, alpha, moments, median_contrib) is handed over as the first
    elements of a buffer whose next element is a sentinel: 2^30 for contrib, INT_MAX for median_contrib,
    NaN for the float planes.  On the last row the missing pixel's values are those sentinels (on the
    other rows it is the next row's first pixel, which both calls read alike).  A walk that takes the
    missing pixel up, its contrib read together with any other of its planes, turns the rows non-finite;
    the rows must instead equal those of plain planes, up to the order of their float atomics.
    What this cannot see: a dropped guard on the geometry reads alone.  The missing pixel's cont is 0,
    and cont gates every use of its gdist, gmed, A, D, D2 and median record, so such reads leave the
    rows unchanged."""
    o = ops()
    sc = random_scene(400, 97, 61, 4, cam="posed_a", seed=97, spread=1.1)
    H, W = 61, 97
    res = geo_frame(sc, 1.5, 20.0)
    args = bwd_args(res)
    up = [T(a.astype(np.float32)) for a in upstream6(H, W, 7)]
    assert (n(res[1][1])[-1, -1] > 0) and W % 2 == 1   # the last row's last pixel is drawn

    def tail(t, bad):
        buf = torch.full((t.numel() + 1,), bad, dtype=t.dtype, device=DEV)
        buf[:-1] = t.reshape(-1)
        return buf[:-1].reshape(t.shape)

    ref = n(o.splatB_surfel_geometry(H, W, *args, *up, near=1.5, far=20.0))
    nan = float("nan")
    a = [args[0], tail(args[1], 2 ** 30), tail(args[2], nan), args[3], args[4], tail(args[5], nan),
         tail(args[6], nan), tail(args[7], 2 ** 31 - 1)]
    got = n(o.splatB_surfel_geometry(H, W, *a, *[tail(u, nan) for u in up], near=1.5, far=20.0))
    assert np.isfinite(got).all()
    assert np.abs(got - ref).max() <= 1e-5 * np.abs(ref).max()


# ---------------------------------------------------------------- 2. median ties
def test_median_ties_exactly():
    """the tie stacks: at every centre median_contrib is the model's strict tau > 0.5 choice, with no
    margin; median_depth is that record's hit depth; dL/dmedian at one centre only (every other upstream
    plane None) gives exactly one nonzero row, the median record's"""
    o = ops()
    sc, medc, tie = tie_stacks()
    H, W = sc["H"], sc["W"]
    res = geo_frame(sc)
    g, out = res
    pre = pre_of(sc)
    bins = so.bin_f32(H, W, pre)
    assert np.array_equal(n(out[3]), bins[1]) and np.array_equal(n(out[4]), bins[2])
    rp = record_pre(pre, n(g[4]))
    fwd = sg.render_geometry(H, W, rp, sc["alphas"], bins, exact=True)
    ys, xs = tie_claims(sc, rp, bins, fwd, medc, tie)   # the kernels' own records reach the ties too
    dist, med, mom, mc = (n(x) for x in out[8:])
    assert np.array_equal(mc[ys, xs], medc)
    assert (mc == fwd["median_contrib"])[~fwd["ambiguous"]].all()
    mrec = medc - 1 + TIE_LEN * np.arange(len(medc))
    assert (np.abs(med[ys, xs] - rp["M"][mrec, 2, 2]) <= 1e-4 * max(1.0, np.abs(fwd["median_depth"]).max())).all()
    for t, (y, x) in enumerate(zip(ys, xs)):
        dlm = torch.zeros((H, W), device=DEV)
        dlm[y, x] = 1.0
        rows = n(o.splatB_surfel_geometry(H, W, *bwd_args(res), dloss_dmedian=dlm))
        nz = np.flatnonzero(np.abs(rows).max(axis=1) > 0)
        assert list(nz) == [mrec[t]], (t, list(nz))


# ---------------------------------------------------------------- 3. dead tiles
def test_geometry_dead_tiles_at_4k_and_1km():
    """far = 100: the live hits at about 1 km have m > 1; the dead tiles have every geometry plane
    exactly 0, and every row and gradient of a dead surfel is exactly 0 with all six upstream planes"""
    o = ops()
    sc, dead = dead_scene()
    H, W = DEAD_H, DEAD_W
    res = geo_frame(sc, 0.2, 100.0)
    g, out = res
    bins = so.bin_f32(H, W, pre_of(sc))
    assert np.array_equal(n(out[3]), bins[1])
    dpx = tile_map(H, W, dead_claims(sc, dead, bins).reshape(-1))
    dist, med, mom, medc = (n(x) for x in out[8:])
    alpha, contrib = n(out[6]), n(out[1])
    for p in (dist, med, medc):
        assert not p[dpx].any()
    assert not mom[:, dpx].any()
    live = contrib > 0
    assert live.sum() > 20000 and (mom[0][live] > alpha[live]).all() and (medc[live] > 0).all()
    up = [T(a.astype(np.float32)) for a in upstream6(H, W, 5)]
    rows = o.splatB_surfel_geometry(H, W, *bwd_args(res), *up)
    P = params(sc)
    gr = o.surfel_preprocessB(P["pws"], P["rots"], P["scales"], P["shs"], P["Rcw"], P["tcw"], P["twc"], *cam_args(sc),
                              rows)
    assert dead.sum() > 10000
    assert not n(rows)[dead].any() and n(rows)[~dead].any()
    for x in gr:
        assert not n(x).reshape(len(dead), -1)[dead].any()


# ---------------------------------------------------------------- 4. poisoned allocations
@pytest.mark.parametrize("W,H", [(160, 96), (97, 61), (17, 9), (7, 5)])
def test_geometry_empty_tiles_over_poisoned_memory(W, H):
    """the geometry frame's planes allocated over memory filled with 0x7f7f7f7f: distortion, both
    moments, median_depth and median_contrib (and the surfel planes) exactly 0 and finite on tiles
    without patches; the exact path, the exact path learning the capacity bounds and the capacity path
    bit-identical.  7x5 is one tile: rendered once with content, once with every surfel culled."""
    o = ops()
    sc = random_scene(60, W, H, 1, cam="posed_a", seed=W + H, spread=0.25)
    g = gpu_preprocess(sc)
    bins = so.bin_f32(H, W, pre_of(sc))
    live = bins[1][:, 1] > bins[1][:, 0]
    gx, gy = (W + 15) // 16, (H + 15) // 16
    assert live.any() and (gx * gy == 1 or (~live).any())
    cases = [(g[1], live)]
    if W * H < 64:
        cases.append((torch.full_like(g[1], -1.0), np.zeros_like(live)))
    for depths, lv in cases:
        o._CAPACITY.pop(("surfel", torch.device(DEV).index or 0, H, W, len(sc["pws"])), None)
        outs = []
        for capacity in (False, True, True):   # exact; exact learning the bounds; the capacity path
            poison(3 * H * W)
            outs.append(o.splat_surfel_geometry(H, W, g[0], depths.clone(), g[2].clone(), g[4], 0.3, 30.0,
                                                capacity=capacity))
            torch.cuda.synchronize()
        empty = ~tile_map(H, W, lv)
        for out in outs:
            image, contrib, ftau, _, _, depth, alpha, normal, dist, med, mom, medc = [n(x) for x in out]
            for p in (image, normal, mom):
                assert np.isfinite(p).all() and not p[:, empty].any()
            for p in (depth, alpha, ftau, dist, med):
                assert np.isfinite(p).all() and not p[empty].any()
            assert not contrib[empty].any() and not medc[empty].any()
            if lv.any():
                assert alpha[~empty].max() > 0 and mom[0][~empty].max() > 0
            for x, y in zip(outs[0], out):
                assert torch.equal(x, y)


# ---------------------------------------------------------------- 5. capacity path, backward
def test_geometry_capacity_path_backward():
    """rows and parameter gradients of a capacity-path frame with both geometry gradients set: the
    exact path's up to the order of their float atomics"""
    o = ops()
    sc = random_scene(2000, 203, 121, 4, cam="posed_b", seed=12, spread=1.1)
    H, W = sc["H"], sc["W"]
    up = [T(a.astype(np.float32)) for a in upstream6(H, W, 12)]
    P = params(sc)

    def grads(capacity):
        res = geo_frame(sc, 0.3, 30.0, capacity=capacity)
        rows = o.splatB_surfel_geometry(H, W, *bwd_args(res), *up, near=0.3, far=30.0)
        gr = o.surfel_preprocessB(P["pws"], P["rots"], P["scales"], P["shs"], P["Rcw"], P["tcw"], P["twc"],
                                  *cam_args(sc), rows)
        return res[1], [n(rows)] + [n(x) for x in gr]

    o._CAPACITY.clear()
    out_e, exact = grads(False)
    grads(True)   # exact, learns the bounds
    frames = o.CAPACITY_STATS["capacity_frames"]
    out_c, cap = grads(True)
    assert o.CAPACITY_STATS["capacity_frames"] == frames + 1
    for a, b in zip(out_e, out_c):
        assert torch.equal(a, b)
    for a, b in zip(exact, cap):
        assert np.abs(a).max() > 0 and np.abs(a - b).max() <= 1e-5 * np.abs(a).max()


# ---------------------------------------------------------------- 6. GSFunctionSurfelGeometry
def camera_of(sc):
    from easygaussiansplatting_b200.gsfunction import Camera
    return Camera(sc["W"], sc["H"], sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(sc["Rcw"]), T(sc["tcw"]), T(sc["twc"]))


def leaves_of(sc):
    P = {k: T(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    al = T(sc["alphas"][:, None]).requires_grad_()
    us = torch.zeros((len(sc["pws"]), 2), device=DEV, requires_grad=True)
    return [P["pws"], P["shs"], al, P["scales"], P["rots"], us]


def apply_geometry(sc, leaves, *nf):
    from easygaussiansplatting_b200.gsfunction import GSFunctionSurfelGeometry
    return GSFunctionSurfelGeometry.apply(*leaves, camera_of(sc), *nf)


def ops_chain(sc, planes, near=0.2, far=100.0):
    """splat_surfel_geometry, splatB_surfel_geometry on `planes` (six, None = not read) and
    surfel_preprocessB -> ((pws, shs, alphas, scales, rots, us) gradients in the leaves' order, rows)"""
    o = ops()
    H, W = sc["H"], sc["W"]
    res = geo_frame(sc, near, far)
    rows = o.splatB_surfel_geometry(H, W, *bwd_args(res), *planes, near=near, far=far)
    P = params(sc)
    d = o.surfel_preprocessB(P["pws"], P["rots"], P["scales"], P["shs"], P["Rcw"], P["tcw"], P["twc"], *cam_args(sc),
                             rows)
    return [d[0], d[1], d[2], d[3], d[4], d[5]], rows


def same_to_atomics(sc, got, chain):
    """the leaves' gradients against the ops chain's, per surfel.  Both run the same kernels on the same
    planes, so their rows differ only in the order of their float atomics, and surfel_preprocessB maps
    them through the surfel's K^T and frame alike: within the 1e-5 of the capacity-path comparison,
    taken per surfel of max(its gradient norm, 1e-3 |K| |row|).  The second term is check_rows' floor:
    a median-only loss reaches pws, scales and rots through M's third row alone, whose K^T terms cancel
    to 1e-4 of their size, so the rows' last-bit differences reach those gradients at the size of the
    terms, not of the result."""
    want, rows = chain
    N = len(sc["pws"])
    a = np.concatenate([n(x).reshape(N, -1) for x in got], 1).astype(np.float64)
    b = np.concatenate([n(x).reshape(N, -1) for x in want], 1).astype(np.float64)
    K = np.array([[sc["fx"], 0, sc["cx"]], [0, sc["fy"], sc["cy"]], [0, 0, 1.0]])
    norm = np.maximum(np.linalg.norm(b, axis=1), 1e-3 * np.abs(K).sum() * np.linalg.norm(n(rows), axis=1))
    err = np.abs(a - b).max(axis=1)
    assert (err <= 1e-5 * norm + 1e-30).all(), float((err / (norm + 1e-30)).max())
    assert np.abs(b).max() > 0


@pytest.mark.parametrize("loss", ["dist_mean", "median_t", "dist_and_median"])
def test_gsfunction_geometry_upstream_views(loss):
    """one-output losses and the views autograd hands the backward (the stride-0 expand of
    distortion.mean(), median.t()): the gradients of the same planes passed as contiguous tensors"""
    sc = random_scene(900, 96, 64, 16, cam="posed_a", seed=19, spread=1.1, z=(1.0, 6.0))
    H, W = sc["H"], sc["W"]
    leaves = leaves_of(sc)
    outs = apply_geometry(sc, leaves, 0.5, 20.0)
    dist, median = outs[4], outs[5]
    rng = np.random.default_rng(6)
    none4 = [None] * 4
    if loss == "dist_mean":
        scalar, planes = dist.mean(), none4 + [torch.full((H, W), 1.0 / (H * W), device=DEV), None]
    elif loss == "median_t":
        wt = T(rng.normal(size=(W, H)).astype(np.float32))
        scalar, planes = (median.t() * wt).sum(), none4 + [None, wt.t().contiguous()]
    else:
        w1, w2 = (T(rng.normal(size=(H, W)).astype(np.float32)) for _ in range(2))
        scalar, planes = (dist * w1).sum() + (median * w2).sum(), none4 + [w1, w2]
    scalar.backward()
    got = [x.grad for x in leaves]
    got[2] = got[2].reshape(-1)
    same_to_atomics(sc, got, ops_chain(sc, planes, 0.5, 20.0))
    assert np.abs(n(got[0])).max() > 0


def test_gsfunction_geometry_near_far_reach_the_backward():
    """at near = 1.5, far = 20 (hits on both sides of near) dL/dalpha and dL/dus, the rows' entries 9
    and 16-17, match the model's rows at those values per entry (rows_bound), and differ from the
    model's rows at the defaults (the forward's planes, the backward's m at near = 0.2, far = 100) by
    more than ten times that bound"""
    sc = random_scene(500, 96, 64, 4, cam="posed_a", seed=3, spread=1.1, z=(1.0, 6.0))
    H, W = sc["H"], sc["W"]
    near, far = 1.5, 20.0
    g = gpu_preprocess(sc)
    pre = pre_of(sc)
    bins = so.bin_f32(H, W, pre)
    rp = record_pre(pre, n(g[4]))
    fwd = sg.render_geometry(H, W, rp, sc["alphas"], bins, near, far)
    fwd_d = sg.render_geometry(H, W, rp, sc["alphas"], bins)
    ok = ~(fwd["ambiguous"] | fwd_d["ambiguous"])
    z = pre["depths"]
    assert (z[z > 0] < near).any() and (z > near).any()
    rng = np.random.default_rng(8)
    w1, w2 = np.where(ok, rng.normal(size=(H, W)) * 10, 0.0), np.where(ok, rng.normal(size=(H, W)), 0.0)
    leaves = leaves_of(sc)
    outs = apply_geometry(sc, leaves, near, far)
    ((outs[4] * T(w1.astype(np.float32))).sum() + (outs[5] * T(w2.astype(np.float32))).sum()).backward()
    got = np.concatenate([n(leaves[2].grad).reshape(-1, 1), n(leaves[5].grad)], 1)
    cols = [9, 16, 17]
    want, ab = sg.render_backward_geometry(H, W, rp, sc["alphas"], bins, fwd, dl_distortion=w1, dl_median=w2,
                                           near=near, far=far, abs_rows=True)
    rows_bound(got, want[:, cols], ab[:, cols], "near/far")
    other, ab_d = sg.render_backward_geometry(H, W, rp, sc["alphas"], bins, fwd, dl_distortion=w1, dl_median=w2,
                                              abs_rows=True)
    floor = 1e-9 * ab[:, cols].max(axis=0)[None, :] + 1e-30
    assert (np.abs(got - other[:, cols]) / (1e-4 * ab[:, cols] + floor)).max() > 10


def test_2dgs_loss_through_autograd():
    """L = gau_loss(image, gt) + 100 distortion.mean() + 0.05 (1 - (normal . depth_to_normal(median)
    alpha.detach())).mean(): the upstream planes autograd hands the class, captured with tensor hooks;
    the class's gradients equal the ops chain on them (to the order of the float atomics); the model's
    rows on them match the kernels' rows per surfel within rows_bound, except rows with a record
    composited at a pixel the model flags ambiguous (5e-3 of the entry's absolute sum), under 1 % of
    the live rows"""
    from easygaussiansplatting_b200.loss import depth_to_normal, gau_loss
    # small surfels (2.2 records per pixel): few rows share a pixel with an ambiguous threshold
    sc = random_scene(900, 96, 64, 4, cam="posed_b", seed=29, spread=1.1, z=(1.0, 6.0), size=(0.003, 0.02),
                      alpha=(0.3, 0.95))
    H, W = sc["H"], sc["W"]
    leaves = leaves_of(sc)
    image, depth, alpha, normal, dist, median, _ = apply_geometry(sc, leaves)
    cap = {}
    for name, t in (("image", image), ("normal", normal), ("distortion", dist), ("median", median)):
        t.register_hook(lambda gr, name=name: cap.__setitem__(name, gr.detach().contiguous().clone()))
    gt = T(np.random.default_rng(2).uniform(size=(3, H, W)).astype(np.float32))
    ln = (1 - (normal * depth_to_normal(median, camera_of(sc)) * alpha.detach()).sum(0)).mean()
    loss = gau_loss(image, gt) + 100.0 * dist.mean() + 0.05 * ln
    loss.backward()
    assert sorted(cap) == ["distortion", "image", "median", "normal"]
    assert all(n(v).any() for v in cap.values())
    planes = [cap["image"], None, None, cap["normal"], cap["distortion"], cap["median"]]
    got = [x.grad for x in leaves]
    got[2] = got[2].reshape(-1)
    same_to_atomics(sc, got, ops_chain(sc, planes))
    # the model on the same planes, from the kernels' records
    o = ops()
    res = geo_frame(sc)
    rows = n(o.splatB_surfel_geometry(H, W, *bwd_args(res), *planes))
    pre = pre_of(sc)
    bins = so.bin_f32(H, W, pre)
    rp = record_pre(pre, n(res[0][4]))
    fwd = sg.render_geometry(H, W, rp, sc["alphas"], bins)
    dl = [None if p is None else n(p).astype(np.float64) for p in planes]
    want, ab = sg.render_backward_geometry(H, W, rp, sc["alphas"], bins, fwd, *dl, abs_rows=True)
    floor = 1e-9 * ab.max(axis=0)[None, :] + 1e-30
    ratio = (np.abs(rows.astype(np.float64) - want) / (1e-4 * ab + floor)).max(axis=1)
    flagged = sg.composited_at(H, W, rp, sc["alphas"], bins, fwd, fwd["ambiguous"])
    live = ab.max(axis=1) > 0
    assert live.sum() > 300
    assert ratio[live & ~flagged].max() <= 1.0, float(ratio[live & ~flagged].max())
    assert ratio[flagged].max(initial=0) <= 50.0
    assert flagged.sum() < 0.01 * live.sum(), (int(flagged.sum()), int(live.sum()))
