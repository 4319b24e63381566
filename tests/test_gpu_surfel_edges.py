"""The surfel path (surfel.cu, surfel_math.h, GSFunctionSurfel) against the fp64 oracle binned
independently, at posed cameras and at the rasterizer edges the colour and RGB-D paths are tested at.
Scenes and their oracle-only claims: tests/test_surfel_edge_scenes_cpu.py.

1. Per-surfel outputs of k_surfel_fwd (us, depths, areas, colours, the 80-byte records) against the
   oracle's `preprocess` at the identity and two posed cameras, every SH degree, N at the CTA tails.
2. The oracle binned on its own fp32-rounded (u, depth, area): tile ranges and patch lists equal to
   the kernels'; the four planes, contrib and final_tau on the unambiguous pixels.
3. Gradients in two stages: splatB_surfel's rows against the oracle's rows computed from the
   kernels' own records, per surfel and per entry, within 1e-4 of the entry's sum of absolute
   per-pixel terms; k_surfel_bwd on the kernels' rows against the oracle's `preprocess_backward`,
   per surfel, relative to that surfel's gradient norm.
4. Edge scenes: chunk and list-length edges, early termination, the clamp, tiny alphas, an odd
   frame width with content in its partial tile, a dense scene, edge-on / grazing / sub-pixel /
   needle / frame-sized / off-screen surfels, +-inf cull boxes, the 2^24 area cap, odd frames,
   and 4K dead tiles at 1 km.
5. Every non-empty subset of upstream planes (None, explicit zeros and the oracle agree), and
   GSFunctionSurfel receiving the views autograd hands it.
6. Frames whose planes come from poisoned allocator memory: exactly 0 on tiles without patches,
   on the exact and the capacity path."""
import numpy as np
import pytest
import torch

from oracle import surfel_oracle as so
from test_surfel_edge_scenes_cpu import (CAMERAS, DEAD_H, DEAD_W, composited_pairs, cull_box, dead_claims,
                                         dead_scene, dense_claims, dense_scene, margins, random_scene, special_claims,
                                         special_scene, stack_claims, stack_scene)

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
K3S = (1, 4, 9, 16)


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def n(t):
    return t.detach().cpu().numpy()


def ops():
    from easygaussiansplatting_b200 import ops as o
    return o


def cam_args(sc):
    return (sc["fx"], sc["fy"], sc["cx"], sc["cy"], sc["W"], sc["H"])


def params(sc):
    return {k: T(sc[k]) for k in ("pws", "rots", "scales", "shs", "alphas", "Rcw", "tcw", "twc")}


def gpu_preprocess(sc):
    P = params(sc)
    return ops().surfel_preprocess(P["pws"], P["rots"], P["scales"], P["shs"], P["alphas"], P["Rcw"], P["tcw"],
                                   P["twc"], *cam_args(sc))


def pre_of(sc):
    return so.preprocess(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                         sc["fy"], sc["cx"], sc["cy"])


def with_culled(sc, every=37):
    """every `every`-th surfel moved to camera depth 0.15 (culled: pc.z < 0.2)"""
    Rcw, tcw = np.asarray(sc["Rcw"], np.float64), np.asarray(sc["tcw"], np.float64)
    pc = np.asarray(sc["pws"], np.float64) @ Rcw.T + tcw
    pc[::every, 2] = 0.15
    sc = dict(sc)
    sc["pws"] = np.ascontiguousarray((pc - tcw) @ Rcw, dtype=np.float32)
    return sc


# ---------------------------------------------------------------- 1. per-surfel outputs
def check_preprocess(sc, g=None, pre=None):
    """k_surfel_fwd's outputs against the oracle's preprocess.  Bounds (fp32, u = 2^-24):
    pc carries at most a few roundings of s = |Rcw| |pw| + |tcw|, so depth within 2^-21 (s_z + z),
    u within 2^-20 (f (s_x + |x| s_z / z) / z + |u|); M entries within 2^-19 of |K| [s0 | s1 | |pc| + s]
    (the unit axes R e0, R e1 carry their roundings in every component);
    the colour within 2^-20 (1 + sum |sh|); the unit normal within 1e-6; alpha, u and the colour in
    the record are the very values written to alphas, us and colors.  The cull half-extents lie
    between the fp64 box at the level t = 2 ln(alpha / 0.002) and 1.001 box' + 0.1 px (+ 1e-5 box'
    + 2^-18 (|u| + |c|): row k - u_k m3 rounds at the size of (|u| + |c|) pc.z, c = (cx, cy)), box' the fp64 box at the kernels' level t + 1e-3.  -> (pre, outputs)"""
    pre = pre_of(sc) if pre is None else pre
    us, depths, areas, colors, recs = [n(x) for x in (gpu_preprocess(sc) if g is None else g)]
    N = len(sc["pws"])
    keep = pre["keep"]
    Rcw, tcw = np.asarray(sc["Rcw"], np.float64), np.asarray(sc["tcw"], np.float64)
    s = np.abs(np.asarray(sc["pws"], np.float64)) @ np.abs(Rcw).T + np.abs(tcw)
    pc, z = pre["pc"], np.where(keep, pre["pc"][:, 2], 1.0)
    # culled rows: exactly depth -1, areas 0, u 0, a record that never draws
    assert (depths[~keep] == -1).all() and (areas[~keep] == 0).all() and (us[~keep] == 0).all()
    assert np.isneginf(recs[~keep, 12:14]).all()
    assert (depths[keep] > 0).all()
    k = keep
    assert (np.abs(depths[k] - pc[k, 2]) <= 2.0 ** -21 * (s[k, 2] + z[k])).all()
    for c, f in ((0, sc["fx"]), (1, sc["fy"])):
        b = 2.0 ** -20 * (f * (s[k, c] + np.abs(pc[k, c]) * s[k, 2] / z[k]) / z[k] + np.abs(pre["u"][k, c]))
        err = np.abs(us[k, c] - pre["u"][k, c])
        assert (err <= b).all(), ("u", c, (err / b).max())
    # exact where the footprint is well conditioned.  Two cases are not: a half-extent of millions
    # of pixels below the cap (a disk grazing the camera plane: D / pc.z^2 ~ 1e-6) carries fp32's
    # relative error in D, and sf::footprint's half^2 = centre^2 - (...) / D cancels two terms of
    # size u^2, so its fp32 error grows as |u|^2 2^-24 (about 1 px^2 at u ~ 4000 px, a 4K frame)
    e = pre["ext"]
    tol = 2.0 ** -20 * (np.abs(pre["u"]) + e) ** 2 / np.maximum(e, 1.0)   # |d half| ~ |d half^2| / (2 half)
    well = ((e < 1e5) | (e >= 1.01 * so.AREA_CAP)) & (np.abs(e - np.round(e)) > tol)
    assert np.array_equal(areas[k][well[k]], pre["areas"][k][well[k]])
    assert (np.abs(areas[k] - pre["areas"][k]) <= np.maximum(1, 0.1 * pre["areas"][k])).all()
    shs = np.abs(np.asarray(sc["shs"], np.float64)).reshape(N, -1, 3).sum(1)
    err = np.abs(colors - pre["colors"])
    assert (err <= 2.0 ** -20 * (1 + shs)).all(), (err / (1 + shs)).max()
    # records
    K = np.abs(pre["K"])
    one = np.ones((N, 3))
    cols = np.stack([pre["scales"][:, 0:1] * one, pre["scales"][:, 1:2] * one, np.abs(pc) + s], 2)
    X = np.einsum("ij,njk->nik", K, cols)
    errM = np.abs(recs[:, :9].reshape(N, 3, 3) - pre["M"])
    assert (errM[k] <= 2.0 ** -19 * X[k] + 1e-30).all(), (errM[k] / (X[k] + 1e-30)).max()
    assert np.array_equal(recs[k, 9], np.asarray(sc["alphas"], np.float32)[k])
    assert np.array_equal(recs[k, 10:12], us[k]) and np.array_equal(recs[k, 14:17], colors[k])
    assert (np.abs(recs[k, 17:20] - pre["n"][k]) <= 1e-6).all()
    box = cull_box(pre, sc["alphas"])
    rc = recs[:, 12:14].astype(np.float64)
    ninf = np.asarray(sc["alphas"], np.float32) < np.float32(0.002)
    assert np.array_equal(np.isneginf(rc[k]), np.repeat(ninf[k, None], 2, 1))
    assert np.array_equal(np.isposinf(rc[k]), np.isposinf(box[k]))
    fin = k[:, None] & np.isfinite(box)
    assert (rc[fin] >= box[fin]).all(), (box[fin] - rc[fin]).max()
    top = cull_box(pre, sc["alphas"], dt=1e-3)   # the kernels' level: t + 1e-3
    hi = 1.001 * top[fin] + 0.1 + 1e-5 * top[fin] + 2.0 ** -18 * (np.abs(pre["u"]) + np.abs([sc["cx"], sc["cy"]]))[fin]
    assert (rc[fin] <= hi).all(), (rc[fin] - hi).max()
    return pre, (us, depths, areas, colors, recs)


@pytest.mark.parametrize("k3", K3S)
@pytest.mark.parametrize("cam", list(CAMERAS))
def test_per_surfel_outputs_match_preprocess(cam, k3):
    for N in (1, 127, 128, 129, 20001):
        sc = random_scene(N, 160, 96, k3, cam=cam, seed=N + k3, alpha=(0.0005, 0.999))
        if N > 1:
            sc = with_culled(sc)
        pre, _ = check_preprocess(sc)
        if N > 1:
            assert (~pre["keep"]).any() and pre["keep"].any()
        if N == 20001:
            assert (np.asarray(sc["alphas"]) < 0.002).any()


# ---------------------------------------------------------------- 2. + 3. frames against the oracle
def record_pre(pre, recs):
    """the oracle's per-surfel state with M, u, colour and n taken from the kernels' records: the
    rasterizers compared on their own inputs"""
    r = recs.astype(np.float64)
    p = dict(pre)
    p["M"] = r[:, :9].reshape(-1, 3, 3)
    p["u"], p["colors"], p["n"] = r[:, 10:12], r[:, 14:17], r[:, 17:20]
    return p


def upstream(H, W, seed):
    rng = np.random.default_rng(seed)
    return [rng.normal(size=s) for s in ((3, H, W), (H, W), (H, W), (3, H, W))]


def tile_map(H, W, per_tile):
    gx, gy = (W + 15) // 16, (H + 15) // 16
    return np.repeat(np.repeat(np.asarray(per_tile).reshape(gy, gx), 16, axis=0), 16, axis=1)[:H, :W]


def check_frame(sc, seed=0, claims=None, planes=(True, True, True, True), tiles=None, grads=True):
    """one frame end to end against the oracle binned on its own fp32 (u, depth, area).
    tiles: compare the planes only on these tiles (the oracle renders only them).
    -> dict(out, rows, grads, ref, pre, fwd, amb, bins)"""
    H, W = sc["H"], sc["W"]
    o = ops()
    g = gpu_preprocess(sc)
    pre, (us, depths, areas, colors, recs) = check_preprocess(sc, g)
    bins = so.bin_f32(H, W, pre)
    margins(sc, pre, bins)
    out = o.splat_surfel(H, W, g[0], g[1], g[2], g[4])
    image, contrib, ftau, ranges, gsid, depth, alpha, normal = [n(x) for x in out]
    assert np.array_equal(ranges, bins[1]) and np.array_equal(gsid, bins[2])
    rbins = bins
    if tiles is not None:
        r = bins[1].copy()
        sel = np.zeros(len(r), bool)
        sel[tiles] = True
        r[~sel] = 0
        rbins = (bins[0], r, bins[2], bins[3])
    rp = record_pre(pre, recs)
    fwd = so.render(H, W, rp, sc["alphas"], rbins)
    ref = so.render(H, W, pre, sc["alphas"], rbins)
    live = tile_map(H, W, (bins[1][:, 1] > bins[1][:, 0]))
    sel_px = np.ones((H, W), bool) if tiles is None else tile_map(H, W, np.isin(np.arange(len(bins[1])), tiles))
    amb = fwd["ambiguous"] | ref["ambiguous"]
    ok = ~amb & sel_px
    assert ok.mean() > 0.5 * sel_px.mean()
    if claims is not None:
        claims(pre, bins, ref)
    # planes of the fp64 model (fp32 M, u: the same 1e-4 as test_gpu_surfel.py)
    for name, got, want in (("image", image, ref["image"]), ("normal", normal, ref["normal"])):
        assert np.abs(got - want).max(axis=0)[ok].max(initial=0) < 1e-4, name
    assert np.abs(alpha - ref["alpha"])[ok].max(initial=0) < 1e-4
    assert np.abs(depth - ref["depth"])[ok].max(initial=0) < 1e-4 * max(1.0, np.abs(ref["depth"]).max())
    assert (contrib == ref["contrib"])[ok].all()
    assert np.abs(ftau - ref["final_tau"])[ok].max(initial=0) < 1e-4
    # final_tau is 0 on empty tiles; A + tau = 1 within four roundings per composited record
    assert not ftau[~live].any() and not contrib[~live].any()
    r = np.abs(alpha.astype(np.float64) - (1 - ftau.astype(np.float64))) / (2.0 ** -22 * contrib + 2.0 ** -24)
    assert r[live].max(initial=0) <= 1.0, r[live].max()
    res = dict(out=out, pre=pre, fwd=fwd, amb=amb, bins=bins, g=g, rp=rp, rbins=rbins, ok=ok)
    if grads:
        dl = [np.where(ok, d, 0.0) if use else None for d, use in zip(upstream(H, W, seed), planes)]
        res.update(check_grads(sc, res, dl))
    return res


def rows_bound(got, want, ab, what):
    """|rows - oracle| <= 1e-4 (the entry's absolute sum) + 1e-9 max(absolute sums of its column)"""
    floor = 1e-9 * ab.max(axis=0, initial=0)[None, :] + 1e-30
    err = np.abs(got.astype(np.float64) - want)
    ratio = err / (1e-4 * ab + floor)
    assert ratio.max(initial=0) <= 1.0, (what, float(ratio.max()), np.unravel_index(ratio.argmax(), ratio.shape))


def check_grads(sc, res, dl):
    H, W = sc["H"], sc["W"]
    o = ops()
    out, g = res["out"], res["g"]
    t = [None if d is None else T(d.astype(np.float32)) for d in dl]
    rows = o.splatB_surfel(H, W, g[4], out[1], out[2], out[3], out[4], *t)
    want, ab = so.render_backward(H, W, res["rp"], sc["alphas"], res["rbins"], res["fwd"], *dl, abs_rows=True)
    rows_n = n(rows)
    if res["rbins"] is res["bins"]:
        rows_bound(rows_n, want, ab, "rows")
    # k_surfel_bwd on the kernels' own rows
    P = params(sc)
    gr = o.surfel_preprocessB(P["pws"], P["rots"], P["scales"], P["shs"], P["Rcw"], P["tcw"], P["twc"],
                              *cam_args(sc), rows)
    ref = so.preprocess_backward(res["pre"], rows_n.astype(np.float64))
    names = ("pws", "shs", "alphas", "scales", "rots", "us")
    N = len(sc["pws"])
    got = np.concatenate([n(x).reshape(N, -1) for x in gr], 1).astype(np.float64)
    exp = np.concatenate([ref[k].reshape(N, -1) for k in names], 1)
    # per surfel: relative to its own gradient norm, or to the size of K^T row where that cancels
    K = res["pre"]["K"]
    norm = np.maximum(np.linalg.norm(exp, axis=1), 1e-3 * np.abs(K).sum() * np.linalg.norm(rows_n, axis=1))
    err = np.abs(got - exp).max(axis=1)
    assert (err <= 1e-4 * norm + 1e-30).all(), float((err / (norm + 1e-30)).max())
    assert (n(gr[3])[:, 2] == 0).all()
    return dict(rows=rows_n, grads=dict(zip(names, [n(x) for x in gr])), ref_rows=want, abs_rows=ab)


@pytest.mark.parametrize("cam,k3,N", [("identity", 1, 129), ("posed_a", 4, 700), ("posed_b", 16, 2001),
                                      ("posed_a", 9, 128)])
def test_frames_binned_independently(cam, k3, N):
    sc = random_scene(N, 160, 96, k3, cam=cam, seed=3 * N + k3, spread=1.1)
    res = check_frame(with_culled(sc), seed=N)
    assert np.abs(res["rows"]).max() > 0


# ---------------------------------------------------------------- 4. edge scenes
def test_stack_scene_list_chunk_stop_and_clamp_edges():
    """list lengths 31-33 / 64-65 / 96-97, terminations right after positions 31-33, alpha 0.99,
    nextafter(0.99, 1) and 1.0 at positions 30-33, alphas 0.001 / 0.002, content in the partial
    tile column of an odd-width frame"""
    sc, lens = stack_scene()
    res = check_frame(sc, seed=1, claims=lambda pre, bins, fwd: stack_claims(sc, lens, pre, bins, fwd))
    _, clamped = composited_pairs(sc, res["pre"], res["bins"], res["fwd"])
    assert clamped
    # the alpha-1.0 records, clamped near their centres: dL/dalpha takes no term from a clamped
    # pixel.  The entry-wise bound above is loose here (the absolute sums carry the whole stack
    # behind each record, ~100x the entry); a clamped pixel's term moves these entries by 0.02-0.7 %.
    ones = np.flatnonzero(np.asarray(sc["alphas"]) == 1.0)
    want, got = res["ref_rows"][ones, 9], res["rows"][ones, 9].astype(np.float64)
    assert (np.abs(want) > 0.1).all()
    assert (np.abs(got - want) <= 1e-3 * np.abs(want)).all(), np.abs(got / want - 1).max()


def test_dense_scene_early_termination():
    sc = dense_scene()
    check_frame(sc, seed=2, claims=lambda pre, bins, fwd: dense_claims(bins, fwd))


@pytest.mark.parametrize("cam", ["identity", "posed_b"])
def test_special_surfels(cam):
    """edge-on, grazing, sub-pixel, needle, frame-sized, off-screen, +-inf cull boxes, the 2^24 cap,
    a flipped normal: the capped surfel is drawn, not culled"""
    sc = special_scene(cam=cam)
    res = check_frame(sc, seed=3, claims=lambda pre, bins, fwd: special_claims(sc, pre, bins, fwd,
                                                                                cull_box(pre, sc["alphas"])))
    us, depths, areas, colors, recs = [n(x) for x in res["g"]]
    assert np.isposinf(recs[[6, 8], 12:14]).all() and np.isneginf(recs[7, 12:14]).all()
    assert (areas[8] == so.AREA_CAP).any() and depths[8] > 0
    assert (res["out"][4] == 8).sum().item() >= 0.5 * res["bins"][1].shape[0]
    assert np.abs(res["rows"][8]).max() > 0


@pytest.mark.parametrize("W,H", [(97, 61), (17, 9), (7, 5)])
def test_odd_frames(W, H):
    sc = random_scene(max(40, W * H // 20), W, H, 4, cam="posed_a", seed=W, spread=1.1)
    res = check_frame(sc, seed=W)
    assert (n(res["out"][1])[:, -1] > 0).any()


def test_dead_tiles_at_4k_and_1km():
    """image, depth, alpha and normal exactly 0 on the dead tiles, every gradient of a dead surfel
    exactly 0; the planes against the oracle on a band of tiles"""
    sc, dead = dead_scene()
    H, W = DEAD_H, DEAD_W
    gx = W // 16
    tiles = np.arange(3 * gx)   # the first three tile rows
    res = check_frame(sc, seed=4, tiles=tiles, grads=False)
    dead_t = dead_claims(sc, dead, res["bins"])
    dpx = tile_map(H, W, dead_t.reshape(-1))
    out = [n(x) for x in res["out"]]
    for i in (0, 5, 6, 7):
        p = out[i]
        assert not (p[:, dpx] if p.ndim == 3 else p[dpx]).any(), i
    assert not out[1][dpx].any()
    dl = [d.astype(np.float32) for d in upstream(H, W, 4)]
    o = ops()
    g = res["g"]
    rows = o.splatB_surfel(H, W, g[4], res["out"][1], res["out"][2], res["out"][3], res["out"][4], *[T(d) for d in dl])
    P = params(sc)
    gr = o.surfel_preprocessB(P["pws"], P["rots"], P["scales"], P["shs"], P["Rcw"], P["tcw"], P["twc"],
                              *cam_args(sc), rows)
    assert dead.sum() > 10000
    assert not n(rows)[dead].any()
    for x in gr:
        assert not n(x).reshape(len(dead), -1)[dead].any()
    assert n(rows)[~dead].any()


# ---------------------------------------------------------------- 5. upstream plane subsets and views
SUBSETS = [tuple(bool(m >> b & 1) for b in range(4)) for m in range(1, 16)]


def test_upstream_plane_subsets():
    """each of the 15 non-empty subsets of (image, depth, alpha, normal) with the rest None: the rows
    match the oracle's with zeros for the rest, and the call with explicit zero planes to the
    order of the float atomics"""
    sc = random_scene(600, 64, 48, 16, cam="posed_b", seed=17, spread=1.1)
    res = check_frame(sc, seed=17, grads=False)
    H, W = sc["H"], sc["W"]
    o = ops()
    g, out = res["g"], res["out"]
    full = [np.where(res["ok"], d, 0.0) for d in upstream(H, W, 17)]
    for sub in SUBSETS:
        dl = [d if use else None for d, use in zip(full, sub)]
        rows = n(o.splatB_surfel(H, W, g[4], *out[1:5], *[None if d is None else T(d.astype(np.float32)) for d in dl]))
        want, ab = so.render_backward(H, W, res["rp"], sc["alphas"], res["bins"], res["fwd"], *dl, abs_rows=True)
        rows_bound(rows, want, ab, sub)
        zeros = n(o.splatB_surfel(H, W, g[4], *out[1:5], *[T((d if use else 0 * d).astype(np.float32))
                                                            for d, use in zip(full, sub)]))
        assert (np.abs(rows - zeros) <= 1e-5 * ab + 1e-30).all(), sub


@pytest.mark.parametrize("loss", ["image_sum", "depth_t", "normal_permute", "alpha_mean"])
def test_gsfunction_surfel_upstream_views(loss):
    """one-output losses (autograd passes None for the other planes) and the views it hands the
    backward (the stride-0 expand of .sum(), depth.t(), normal.permute): the gradients of the same
    planes passed as contiguous tensors, to the order of the float atomics"""
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionSurfel
    sc = random_scene(900, 96, 64, 16, cam="posed_a", seed=19, spread=1.1)
    H, W, N = sc["H"], sc["W"], 900
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(sc["Rcw"]), T(sc["tcw"]), T(sc["twc"]))
    P = {k: T(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    al = T(sc["alphas"][:, None]).requires_grad_()
    us = torch.zeros((N, 2), device=DEV, requires_grad=True)
    image, depth, alpha, normal, _ = GSFunctionSurfel.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us, cam)
    rng = np.random.default_rng(5)
    if loss == "image_sum":
        scalar, planes = image.sum(), (torch.ones((3, H, W), device=DEV), None, None, None)
    elif loss == "depth_t":
        wt = T(rng.normal(size=(W, H)).astype(np.float32))
        scalar, planes = (depth.t() * wt).sum(), (None, wt.t().contiguous(), None, None)
    elif loss == "normal_permute":
        wn = T(rng.normal(size=(H, W, 3)).astype(np.float32))
        scalar, planes = (normal.permute(1, 2, 0) * wn).sum(), (None, None, None, wn.permute(2, 0, 1).contiguous())
    else:
        scalar, planes = alpha.mean(), (None, None, torch.full((H, W), 1.0 / (H * W), device=DEV), None)
    scalar.backward()
    got = [P["pws"].grad, P["shs"].grad, al.grad.reshape(-1), P["scales"].grad, P["rots"].grad, us.grad]
    o = ops()
    g = gpu_preprocess(sc)
    out = o.splat_surfel(H, W, g[0], g[1], g[2], g[4])
    rows = o.splatB_surfel(H, W, g[4], *out[1:5], *planes)
    Pp = params(sc)
    want = o.surfel_preprocessB(Pp["pws"], Pp["rots"], Pp["scales"], Pp["shs"], Pp["Rcw"], Pp["tcw"], Pp["twc"],
                                *cam_args(sc), rows)
    for a, b in zip(got, want):
        a, b = n(a).reshape(N, -1), n(b).reshape(N, -1)
        assert np.abs(a - b).max() <= 1e-5 * np.abs(b).max() + 1e-30
    assert np.abs(n(got[0])).max() > 0


# ---------------------------------------------------------------- 6. poisoned allocations
@pytest.mark.parametrize("W,H", [(160, 96), (97, 61), (17, 9), (7, 5)])
def test_empty_tiles_over_poisoned_memory(W, H):
    """planes allocated over memory filled with 0x7f7f7f7f: image, depth, alpha, normal, contrib and
    final_tau exactly 0 on tiles without patches (k_tile_list: 16-byte stores when W % 4 == 0, scalar
    ones otherwise; the normal plane by its own memset), exact and capacity paths bit-identical.
    7x5 is one tile: rendered once with content, once with every surfel culled."""
    from test_gpu_rgbd_edges import poison
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
            outs.append(o.splat_surfel(H, W, g[0], depths.clone(), g[2].clone(), g[4], capacity=capacity))
            torch.cuda.synchronize()
        empty = ~tile_map(H, W, lv)
        for out in outs:
            image, contrib, ftau, _, _, depth, alpha, normal = [n(x) for x in out]
            for p in (image, normal):
                assert np.isfinite(p).all() and not p[:, empty].any()
            for p in (depth, alpha, ftau):
                assert np.isfinite(p).all() and not p[empty].any()
            assert not contrib[empty].any()
            if lv.any():
                assert alpha[~empty].max() > 0
            for x, y in zip(outs[0], out):
                assert torch.equal(x, y)
