"""The RGB-D rasterizer pair (k_draw_rgbd, k_draw_bwd_rgbd) and the depth term of the fused
per-Gaussian backward (k_preprocess_bwd's DEPTH forms) at the edges the colour path is tested at.

1. The colour rasterizers' schedule-edge scenes (test_gpu_parity.py) through `check_rgbd`: patch
   counts at the whole-tile / four-entry and chunk edges, partial phase-B flushes, the clamp shuffle
   path, opaque stacks, dense early termination, the opacity clamp, huge and needle footprints, and
   dead sparse 4K tiles with 1 km depths (64-bit keys).
2. Upstream-gradient edges of k_draw_bwd_rgbd: one upstream plane at a time, pixels of empty tiles
   (the D and A planes of a frame allocated over poisoned memory), and the views autograd hands
   GSFunctionFusedRGBD.
3. preprocessB(..., dloss_ddepths=gz) against the oracle chain at every SH degree and at the CTA
   tails, in the plain and the moment-row form: rows whose only gradient is dL/dz, culled rows,
   and the bit-level contract (gz = 0, offset views, refused arguments).

Tolerances are those of test_gpu_rgbd.py (rasterizer) and test_gpu_fused_oracle.py (chain)."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from oracle import rgbd_oracle as orgbd
from test_gpu_fused_oracle import (K3S, NS, cam_args, edge_scene, finite_rows, moment_case, norm_err, oracle_stages,
                                   params, shifted)
from test_gpu_parity import (BOUNDARY_GX, DEAD_H, DEAD_W, DEV, boundary_frame, boundary_scene, clamp_scene,
                             dead_sparse_scene, dense_scene, gaussians_in_tile, huge_needle_scene, n, op_inputs,
                             scene_with_culls, stage_pipeline, t)
from test_gpu_rgbd import bound, check_rgbd, preprocess, upstream

pytestmark = pytest.mark.gpu


def ops():
    from easygaussiansplatting_b200 import ops as o
    return o


def tile_map(H, W, per_tile):
    """per-tile values [gy * gx] -> [H, W], each pixel its tile's value"""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    return np.repeat(np.repeat(np.asarray(per_tile).reshape(gy, gx), 16, axis=0), 16, axis=1)[:H, :W]


def tile_pixels(a, i, gx):
    """the 16x16 pixels of tile i of a frame gx tiles wide"""
    return a[16 * (i // gx):16 * (i // gx) + 16, 16 * (i % gx):16 * (i % gx) + 16]


def tau_bound_ratio(A, ftau, contrib):
    """|A - (1 - final_tau)| / (2^-22 contrib + 2^-24).  A = sum w and tau = prod (1 - alpha')
    satisfy A + tau = 1 exactly; in fp32 each composited record adds at most four roundings
    (w, the sum, 1 - alpha', tau) of operands <= 1, so the ratio is <= 1 on every pixel of a tile
    with patches"""
    A, ftau = np.asarray(A, np.float64), np.asarray(ftau, np.float64)
    return np.abs(A - (1.0 - ftau)) / (2.0 ** -22 * np.asarray(contrib, np.float64) + 2.0 ** -24)


# ---------------------------------------------------------------- scene claims (also run on the CPU)
def boundary_claims(ref, expect, survivor_tiles, stack_tiles):
    """boundary_scene reaches its edges: patch counts as built, survivors in block 0 only,
    stack tiles composite m + 2 records on every pixel"""
    gx = BOUNDARY_GX
    lens = ref["ranges"][:, 1] - ref["ranges"][:, 0]
    for i, k in expect.items():
        assert lens[i] == k, (i, lens[i], k)
    assert (lens[len(expect):] == 0).all()
    con = ref["contrib"]
    for i, s in survivor_tiles.items():
        blk = tile_pixels(con, i, gx).copy()
        assert blk[:8, :8].max() > 0
        blk[:8, :8] = 0
        assert not blk.any(), "survivors of tile %d reach beyond block 0" % i
    for i, c in stack_tiles.items():
        assert (tile_pixels(con, i, gx) == c).all(), i


def dense_claims(ref):
    """the dense scene: lists over 300 patches, over half the pixels end at tau < 1e-4"""
    lens = ref["ranges"][:, 1] - ref["ranges"][:, 0]
    assert lens.max() > 300 and (ref["final_tau"] < 1e-4).mean() > 0.5
    assert ref["contrib"].max() < lens.max()


def dead_sparse_claims(ref):
    """dead_sparse_scene: 1-3 patches per tile, exactly the checkerboard of alpha-0.0015 tiles
    composites nothing, and the depth keys need the 64-bit layout.  -> dead tiles [gy, gx]"""
    gx, gy = DEAD_W // 16, DEAD_H // 16
    lens = ref["ranges"][:, 1] - ref["ranges"][:, 0]
    assert lens.min() >= 1 and lens.max() <= 3
    dead = ref["contrib"].reshape(gy, 16, gx, 16).max(axis=(1, 3)) == 0
    assert np.array_equal(dead, (np.add.outer(np.arange(gy), np.arange(gx)) % 2) == 1)
    depth_bits = int((ref["keys"] & 0xFFFFFFFF).max()).bit_length()
    tile_bits = (gx * gy - 1).bit_length()
    assert depth_bits >= 20 and tile_bits == 15 and depth_bits + tile_bits > 32
    return dead


# ---------------------------------------------------------------- 1. rasterizer pair at the schedule edges
def test_rgbd_patch_count_and_survivor_boundaries():
    """boundary_scene with a different depth offset per tile in [1, 20] m (the per-record
    dL/dD z term differs between the records of one flush)"""
    parts, expect, survivor_tiles, stack_tiles = boundary_scene(np.random.default_rng(7),
                                                                z0s=np.random.default_rng(70).uniform(1.0, 20.0, 64))
    W, H = boundary_frame(expect)
    out, ref, _ = check_rgbd(H, W, *op_inputs(parts), seed=7, tile_z=True)
    boundary_claims(ref, expect, survivor_tiles, stack_tiles)
    A, ftau, con = n(out[6]), n(out[2]), n(out[1])
    for i in stack_tiles:
        r = tau_bound_ratio(tile_pixels(A, i, BOUNDARY_GX), tile_pixels(ftau, i, BOUNDARY_GX),
                            tile_pixels(con, i, BOUNDARY_GX))
        assert r.max() <= 1.0, (i, r.max())


def test_rgbd_dense_early_termination():
    sc = dense_scene()
    W, H = sc["width"], sc["height"]
    o = stage_pipeline(sc, calc_J=False)
    out, ref, _ = check_rgbd(H, W, o["us"], o["cinv2ds"], t(sc["alphas"]), o["depths"], o["colors"], o["areas"],
                             seed=11)
    dense_claims(ref)
    live = tile_map(H, W, ref["ranges"][:, 1] - ref["ranges"][:, 0]) > 0
    A = n(out[6])
    r = tau_bound_ratio(A, n(out[2]), n(out[1]))
    assert r[live].max(initial=0) <= 1.0, r[live].max()
    assert not A[~live].any()   # (an empty tile keeps tau 0 and A 0)


def test_rgbd_alpha_clamp_and_tiny_alpha():
    sc = clamp_scene()
    W, H = sc["width"], sc["height"]
    o = stage_pipeline(sc, calc_J=False)
    check_rgbd(H, W, o["us"], o["cinv2ds"], t(sc["alphas"]), o["depths"], o["colors"], o["areas"], seed=2)


def test_rgbd_huge_and_needle_gaussians():
    """20x the float bound, for the reason test_splat_huge_and_needle_gaussians gives: the fp32
    Mahalanobis terms of a 100:1 needle cancel from ~1e5 to O(10)"""
    sc = huge_needle_scene()
    W, H = sc["width"], sc["height"]
    o = stage_pipeline(sc, calc_J=False)
    check_rgbd(H, W, o["us"], o["cinv2ds"], t(sc["alphas"]), o["depths"], o["colors"], o["areas"], seed=13,
               tol_scale=20.0)


def test_rgbd_dead_sparse_tiles_and_far_depths():
    """D and A exactly 0 on the dead tiles; every gradient of a dead Gaussian exactly 0, through
    the full call and the moment rows"""
    W, H = DEAD_W, DEAD_H
    parts = dead_sparse_scene(np.random.default_rng(11))
    us, ci, al, d, col, ar = op_inputs(parts)
    out, ref, g5 = check_rgbd(H, W, us, ci, al, d, col, ar, seed=11, tile_z=True)
    dead = dead_sparse_claims(ref)
    dead_px = tile_map(H, W, dead.reshape(-1))
    assert not n(out[5])[dead_px].any() and not n(out[6])[dead_px].any()
    dead_g = np.concatenate([np.full(len(p[0]), dead.reshape(-1)[i]) for i, p in enumerate(parts)])
    assert dead_g.sum() > 10000
    for g in g5:
        assert not n(g).reshape(len(dead_g), -1)[dead_g].any()
    # the moment rows of the same frame
    zmax = max(float(np.abs(ref["z"][ref["gsid"]]).max()), 1.0)
    dl, dld, dla = upstream(W, H, 11, zmax)
    mom, dz = ops().splatB_rgbd(H, W, us, ci, al, d, col, *out[1:5], t(dl), t(dld), t(dla), moments_only=True)
    assert not n(mom)[dead_g].any() and not n(dz)[dead_g].any()
    assert n(dz)[~dead_g].any()


# ---------------------------------------------------------------- 2. upstream-gradient edges of k_draw_bwd_rgbd
def moments_as_grads(mom, ci):
    """raw moment rows -> (dus, dcinv2ds, dalphas, dcolors) in fp64, k_finalize_grads' formulas"""
    m, c = np.asarray(mom, np.float64), np.asarray(ci, np.float64)
    none = (m[:, 0] == 0) & (m[:, 1] == 0)
    with np.errstate(invalid="ignore"):
        du = -np.stack([c[:, 0] * m[:, 0] + c[:, 1] * m[:, 1], c[:, 1] * m[:, 0] + c[:, 2] * m[:, 1]], axis=1)
    du[none] = 0
    dc = np.stack([-0.5 * m[:, 2], -m[:, 3], -0.5 * m[:, 4]], axis=1)
    return du, dc, m[:, 5], m[:, 6:9]


@pytest.mark.parametrize("plane", ["depth", "alpha", "gamma"])
def test_rgbd_backward_one_upstream_plane(plane):
    """only one of dL/dD, dL/dA, dL/dgamma non-zero: the full call and the moment rows against the
    oracle; dL/dz is exactly 0 unless dL/dD is given"""
    o = ops()
    N, W, H = 3000, 979, 546
    sc = scene_with_culls(N, W, H, 3, 31)
    us, ci, col, d, ar = preprocess(sc)
    al = t(sc["alphas"])
    d0, ar0 = n(d).copy(), n(ar).copy()
    out = o.splat_rgbd(H, W, us, ci, al, d, col, ar)
    ref = orgbd.splat_rgbd(H, W, n(us), n(ci), n(al), d0, n(col), ar0)
    assert np.array_equal(n(out[4]), ref["gsid"])
    zmax = max(float(np.abs(ref["z"][ref["gsid"]]).max()), 1.0)
    dl, dld, dla = upstream(W, H, 31, zmax)
    if plane != "gamma":
        dl = np.zeros_like(dl)
    if plane != "depth":
        dld = np.zeros_like(dld)
    if plane != "alpha":
        dla = np.zeros_like(dla)
    full = o.splatB_rgbd(H, W, us, ci, al, d, col, *out[1:5], t(dl), t(dld), t(dla))
    mom, dz = o.splatB_rgbd(H, W, us, ci, al, d, col, *out[1:5], t(dl), t(dld), t(dla), moments_only=True)
    *ref5, amb = orgbd.splat_backward_rgbd(H, W, n(us), n(ci), n(al), n(col), ref["z"], ref, dl, dld, dla,
                                           return_ambiguous=True)
    assert amb.mean() <= 0.01
    names = ("dus", "dcinv2ds", "dalphas", "dcolors")
    for got, want, name in zip(full[:4], ref5[:4], names):
        bound(got, want, amb, name)
    for got, want, name in zip(moments_as_grads(n(mom), n(ci)), ref5[:4], names):
        bound(torch.from_numpy(got), want, amb, "moment rows: " + name)
    if plane == "depth":
        bound(full[4], ref5[4], amb, "ddepths")
        bound(dz, ref5[4], amb, "moment call: ddepths")
    else:
        assert not bool(full[4].any()) and not bool(dz.any())


def poison(plane_elems):
    """fill the caching allocator's free memory with 0x7f7f7f7f (as float: 3.4e38): the large pool
    through one 256 MB block, the small pool (<= 1 MB) through whole 2 MB segments, and blocks of
    the planes' own size.  An output pixel no kernel writes keeps that value."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    fill = lambda k: torch.full((k,), 0x7f7f7f7f, dtype=torch.int32, device=DEV)
    xs = [fill(64 << 20)] + [fill(1 << 18) for _ in range(8)] + [fill(plane_elems) for _ in range(16)]
    torch.cuda.synchronize()
    del xs


def sparse_frame(W, H, frac, rng):
    """Gaussians in about `frac` of the tiles, none in the last tile column and row (partial
    tiles at odd W / H): op-surface inputs and the bool [gy, gx] of tiles that have some"""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    used = np.zeros((gy, gx), bool)
    inner = np.zeros((gy, gx), bool)
    inner[:max(gy - 1, 1), :max(gx - 1, 1)] = True
    used[inner] = rng.random(inner.sum()) < frac
    used[0, 0] = True
    parts = [gaussians_in_tile(tx, ty, int(rng.integers(1, 40)), rng, z0=rng.uniform(1.0, 20.0))
             for ty, tx in zip(*np.nonzero(used))]
    return op_inputs(parts), used


@pytest.mark.parametrize("W,H", [(979, 546), (960, 544), (17, 9), (7, 5)])
def test_rgbd_empty_tiles_over_poisoned_memory(W, H):
    """D and A of a frame whose planes come from poisoned allocator memory: finite everywhere and
    exactly 0 on the tiles without patches (written by k_tile_list: 16-byte stores when W % 4 == 0,
    scalar ones otherwise and on the partial right-hand tiles), exact and through the capacity
    path, which must agree bit for bit.  7x5 is one tile: rendered once with a Gaussian, once with
    every Gaussian culled (P = 0)."""
    o = ops()
    rng = np.random.default_rng(W * H)
    (us, ci, al, d, col, ar), used = sparse_frame(W, H, 0.12, rng)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    if gx * gy > 4:
        assert 1.0 - used.mean() >= 0.8
    cases = [(d, ar, used)]
    if W * H < 64:
        cases.append((torch.full_like(d, -1.0), ar, np.zeros_like(used)))
    for depths, areas, live in cases:
        key = (torch.device(DEV).index or 0, H, W, us.shape[0])
        o._CAPACITY.pop(key, None)
        outs = []
        for capacity in (False, True, True):   # exact; exact learning the capacity; the capacity path
            poison(H * W)
            before = o.CAPACITY_STATS["capacity_frames"]
            outs.append(o.splat_rgbd(H, W, us, ci, al, depths.clone(), col, areas.clone(), capacity=capacity))
            torch.cuda.synchronize()
        assert o.CAPACITY_STATS["capacity_frames"] == before + 1 or not live.any()
        empty_px = ~tile_map(H, W, live.reshape(-1))
        for out in outs:
            D, A = n(out[5]), n(out[6])
            assert np.isfinite(D).all() and np.isfinite(A).all()
            assert not D[empty_px].any() and not A[empty_px].any()
            assert not n(out[0])[:, empty_px].any() and not n(out[2])[empty_px].any()
            if live.any():
                assert A[~empty_px].max() > 0
            for x, y in zip(outs[0], out):
                assert torch.equal(x, y)


@pytest.mark.parametrize("loss", ["depth_sum", "alpha_mean", "depth_t"])
def test_gsfunction_fused_rgbd_upstream_views(loss, monkeypatch):
    """GSFunctionFusedRGBD's backward receiving the views autograd makes -- the stride-0 expand of
    depth.sum(), the scaled expand of alpha.mean(), the transposed gradient of a loss on depth.t()
    -- gives the gradients of the same upstream planes passed as contiguous tensors.  The
    rasterizer backward's moment rows are sums of float atomics (equal only to their ordering),
    so both runs use the first run's rows: the planes reaching splatB_rgbd must be the same
    values, its outputs agree to rounding, and everything after it is bit-identical."""
    from easygaussiansplatting_b200 import ops as O
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFusedRGBD
    N, W, H = 4001, 320, 200
    sc = scene_with_culls(N, W, H, 12, 45)
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]))
    real = O.splatB_rgbd
    seen = []

    def spy(*args, **kw):
        res = real(*args, **kw)
        seen.append((args[11:14], res))
        if len(seen) == 1:
            return res
        for a, b in zip(seen[0][0], args[11:14]):
            assert torch.equal(a.contiguous(), b.contiguous())
        for a, b in zip(seen[0][1], res):
            assert torch.equal(a != 0, b != 0)
            assert float((a - b).abs().max()) <= 1e-5 * float(a.abs().max())
        return [x.clone() for x in seen[0][1]]

    monkeypatch.setattr(O, "splatB_rgbd", spy)
    rng = np.random.default_rng(5)
    wt = t(rng.normal(size=(W, H)).astype(np.float32))
    grads = []
    for materialised in (True, False):
        params = {k: t(sc[k]).requires_grad_(True) for k in ("pws", "shs", "alphas", "scales", "rots")}
        us0 = torch.zeros((N, 2), device=DEV, requires_grad=True)
        image, depth, alpha, _ = GSFunctionFusedRGBD.apply(params["pws"], params["shs"], params["alphas"],
                                                           params["scales"], params["rots"], us0, cam)
        zero = torch.zeros((H, W), device=DEV)
        # (dL/dD, dL/dA) as contiguous planes, and the scalar loss whose autograd gives the same
        if loss == "depth_sum":
            planes, scalar = (torch.ones((H, W), device=DEV), zero), depth.sum()
        elif loss == "alpha_mean":
            planes, scalar = (zero, torch.full((H, W), 1.0 / (H * W), device=DEV)), alpha.mean()
        else:
            planes, scalar = (wt.t().contiguous(), zero), (depth.t() * wt).sum()
        if materialised:
            torch.autograd.backward([image, depth, alpha], [torch.zeros_like(image), *planes])
        else:
            scalar.backward()
        grads.append([x.grad for x in params.values()] + [us0.grad])
    assert len(seen) == 2
    if loss == "depth_t":   # autograd's gradient of depth is the transposed view of wt
        assert not seen[1][0][1].is_contiguous()
    for a, b in zip(*grads):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert float(grads[0][0].abs().max()) > 0


# ---------------------------------------------------------------- 3. depth term of the fused per-Gaussian backward
FORMS = ("plain", "moments")


def depth_case(k3, N, form):
    """edge_scene, the upstream gradients of `form` and a dL/dz on every row (culled rows too),
    of the size of the geometry part of dL/dpws.  About 2 % of the kept rows and one forced row
    get dL/dz only (no dL/du, dL/dconic, dL/dcolor; all-zero moments).
    -> dict(P, cam, up (positional), kw, gz, ref (oracle chain + depth term), ref0 (without it),
    rows (finite, off the z = 0.2 band), culled (by the device, off the band), depth_only)"""
    from easygaussiansplatting_b200 import ops as O
    sc = edge_scene(N, k3, seed=21 if form == "plain" else 23)
    o = oracle_stages(sc)
    P, cam = params(sc), cam_args(sc)
    rng = np.random.default_rng(100 * N + k3 + (50 if form == "moments" else 0))
    band = o["band"]
    d = n(O.preprocess(*P, *cam)[3])
    if form == "plain":
        keep = (o["depths"] > 0) & (d > 0)
        gu = rng.normal(size=(N, 1, 2)).astype(np.float32)
        gci = rng.normal(size=(N, 1, 3)).astype(np.float32) * 10
        gcol = rng.normal(size=(N, 1, 3)).astype(np.float32)
        gu[~keep] = 0; gci[~keep] = 0; gcol[~keep] = 0
    else:
        m, ci, keep_d, _ = moment_case(sc, N, k3, 31 * N + k3)
        keep = keep_d & (o["depths"] > 0)
    cand = np.flatnonzero(keep & ~band)
    depth_only = keep & ~band & (rng.random(N) < 0.02)
    if len(cand):
        depth_only[cand[rng.integers(len(cand))]] = True
    if form == "plain":
        gu[depth_only] = 0; gci[depth_only] = 0; gcol[depth_only] = 0
        gal = np.zeros((N, 1, 1), np.float32)
        ref0 = orc.chain_backward(sc["Rcw"], gu, gci, gal, gcol, *o["J"])
        up, kw = (t(gu), t(gci), t(gcol)), {}
    else:
        m[depth_only] = 0
        md, cd = m.astype(np.float64), ci.astype(np.float64)
        none = (m[:, 0] == 0) & (m[:, 1] == 0)
        with np.errstate(invalid="ignore"):
            gu = -np.stack([cd[:, 0] * md[:, 0] + cd[:, 1] * md[:, 1], cd[:, 1] * md[:, 0] + cd[:, 2] * md[:, 1]],
                           axis=1)
        gu[none] = 0
        gci = np.stack([-0.5 * md[:, 2], -md[:, 3], -0.5 * md[:, 4]], axis=1)
        ref0 = orc.chain_backward(sc["Rcw"], gu[:, None], gci[:, None], md[:, 5:6, None], md[:, None, 6:9], *o["J"])
        up, kw = (None, None, None), dict(moments=t(m), cinv2ds=t(ci))
    fin = finite_rows(ref0)
    geo = np.abs(ref0["pws"][fin & keep & ~depth_only])
    scale = float(np.percentile(geo.max(axis=1), 90)) if geo.size else 1.0
    gz = (rng.normal(size=N) * scale).astype(np.float32)
    ref = dict(ref0)
    ref["pws"] = ref0["pws"] + orgbd.chain_depth(sc["Rcw"], gz, o["depths"])
    return dict(P=P, cam=cam, up=up, kw=kw, gz=gz, ref=ref, ref0=ref0, rows=fin & ~band,
                culled=(d <= 0) & ~band, depth_only=depth_only, Rcw=sc["Rcw"])


def run_depth(c, gz):
    from easygaussiansplatting_b200 import ops as O
    return O.preprocessB(*c["P"], *c["cam"], *c["up"], **c["kw"], dloss_ddepths=gz)


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("k3", K3S)
def test_preprocess_backward_depth_vs_oracle(k3, N, form):
    """dL/dpws = the chain's + dL/dz Rcw[2,:] within 2e-5 normalised; culled rows exactly 0
    although their dL/dz is not"""
    c = depth_case(k3, N, form)
    got = [n(x) for x in run_depth(c, t(c["gz"]))]
    rows, ref = c["rows"], c["ref"]
    assert norm_err(ref["pws"], c["ref0"]["pws"], rows=rows) > 100 * 2e-5   # the depth term is not lost in the bound
    for g, name in zip(got[:4], ("pws", "shs", "scales", "rots")):
        e = norm_err(g, ref[name], rows=rows)
        assert e <= 2e-5, (name, e)
    cu = c["culled"]
    if N >= 64:
        assert cu.any() and (c["gz"][cu] != 0).all()
    for g in got[:4]:
        assert not g.reshape(N, -1)[cu].any()


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("k3", K3S)
def test_preprocess_backward_depth_only_rows(k3, N, form):
    """a kept Gaussian whose only gradient is dL/dz (the `any` gate of pg::backward_one):
    dL/dpws = fl(dL/dz Rcw[2,:]) within one rounding, dL/dsh, dL/dscale, dL/drot exactly 0"""
    c = depth_case(k3, N, form)
    got = [n(x) for x in run_depth(c, t(c["gz"]))]
    rows = c["depth_only"]
    assert rows.any()
    want = c["gz"].astype(np.float64)[:, None] * np.asarray(c["Rcw"], np.float64).reshape(3, 3)[2][None, :]
    err = np.abs(got[0].astype(np.float64) - want)[rows]
    assert np.all(err <= 2.0 ** -24 * np.abs(want[rows])), err.max()
    assert np.abs(got[0][rows]).max() > 0
    for g in got[1:4]:
        assert not g.reshape(N, -1)[rows].any()
    if form == "moments":
        assert not got[4][rows].any() and not got[5][rows].any()


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("k3", K3S)
def test_preprocess_backward_depth_bits_and_refusals(k3, N, form):
    """dL/dz = 0 gives the bits of the call without it; dL/du and dL/dalpha of the moment form do
    not depend on dL/dz; a dloss_ddepths view one float into its storage gives the same bits; a
    short, float64 or host dloss_ddepths is refused before anything is launched"""
    from easygaussiansplatting_b200 import _lib
    c = depth_case(k3, N, form)
    bits = lambda x: x.view(torch.int32)
    base = run_depth(c, None)
    zero = run_depth(c, torch.zeros(N, device=DEV))
    for i, (a, b) in enumerate(zip(base, zero)):
        assert torch.equal(bits(a), bits(b)), ("dL/dz = 0", i)
    gz = t(c["gz"])
    withz = run_depth(c, gz)
    if form == "moments":
        for a, b in zip(base[4:], withz[4:]):
            assert torch.equal(bits(a), bits(b))
    for i, (a, b) in enumerate(zip(withz, run_depth(c, shifted(gz)))):
        assert torch.equal(bits(a), bits(b)), ("offset dloss_ddepths", i)
    lib = _lib.load()
    torch.cuda.synchronize()
    launches = lib.gsb_profile_launches(-1)
    for bad, err in ((gz[:-1], ValueError), (gz.double(), TypeError), (gz.cpu(), ValueError)):
        with pytest.raises(err):
            run_depth(c, bad)
    assert lib.gsb_profile_launches(-1) == launches
