"""Batched 2D Gaussian Splatting (DESIGN 3.25) at its edges, against the fp64 surfel oracles per entry.
test_gpu_surfel_batch.py pins the forward to the single-camera calls bit for bit; this file holds the
backward and the tall frame's binning to oracles that never see a batch.

(a) k_draw_disk_bwd_batch and k_draw_2dgs_bwd_batch: camera c's rows [c N, (c+1) N) against
    `so.render_backward` / `sgo.render_backward_geometry` on the kernels' own records of camera c, within
    1e-4 of each entry's sum of absolute per-pixel terms (test_gpu_surfel_edges.rows_bound), at C = 2 and 5
    with pad rows and columns in every frame, upstream plane subsets, records from the batch forward and
    re-packed from the single-camera calls; at C = 64 the first, the last and a seeded sample of cameras.
(b) k_disk_fwd_batch<K3> and k_disk_bwd_batch<K3> at every SH degree and N = 1, 127, 128, 129, 1000 (the
    CTA tails): every camera's per-surfel outputs against `so.preprocess`, the summed gradients against
    the fp64 sum over cameras of `so.preprocess_backward` on the kernels' rows (relative to each surfel's
    norm), dL/dus[c] the rows' own; pws, rots, scales and shs each a view 4 bytes past a 16-byte boundary
    in turn: the aligned call's bits, forward and backward.
(c) special_scene's surfels degenerate, capped or culled in some cameras and ordinary in others: finite
    gradients, rows per entry, the per-surfel sums against fp64 over the cameras that composite the
    surfel, dL/dus[c] exactly 0 where camera c culled it.
(d) the tall frame at every key plan the 3DGS batch reaches: each camera's tile lists and in-place culls
    bit for bit against `oracle.bin` on the kernels' own u, depths and areas; the capacity path gives the
    exact path's bits, with and without the geometry planes.
(e) the geometry backward across frame boundaries: disks across the bottom edge of every frame and on
    the first row of the next, rows per camera against fp64, and camera c's rows from frame c's upstream
    planes alone (every other frame's zeroed) equal to the full run's within the per-entry bound.

Scene builders and their claims: test_surfel_batch_edges_cpu.py."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from oracle import surfel_oracle as so
import surfel_geometry_oracle as sgo
from easygaussiansplatting_b200 import ops
from easygaussiansplatting_b200.gsfunction import Camera

from test_batch_edges_cpu import key_plan, plan_shape, tall_height, tall_keys
from test_gpu_batch_edges import check_cameras
from test_gpu_fused_oracle import shifted
from test_gpu_surfel_edges import check_preprocess, record_pre
from test_surfel_batch_edges_cpu import (BOUNDARY, PLAN_BATCHES, SPECIAL_KINDS, boundary_batch, depth_key_max, disks,
                                         build, jittered_cameras, plan_batch, special_batch)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WORST = {}  # (kernel, scene) -> the largest |rows - oracle| / bound seen


@pytest.fixture(autouse=True)
def fresh_capacities():
    ops._CAPACITY.clear()
    yield
    ops._CAPACITY.clear()


@pytest.fixture(scope="module", autouse=True)
def report_worst_ratios():
    yield
    for (kernel, scene), r in sorted(WORST.items()):
        print("worst ratio %-22s %-30s %.3e" % (kernel, scene, r))


def t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).to(DEV)


def n(x):
    return x.detach().cpu().numpy()


def same(x, y):
    return x.shape == y.shape and torch.equal(x.view(torch.int32), y.view(torch.int32))


def gpu_cams(cams, W, H):
    return [Camera(W, H, c["fx"], c["fy"], c["cx"], c["cy"], t(c["Rcw"]), t(c["tcw"]), t(c["twc"])) for c in cams]


def gpu_scene(s):
    return {k: t(s[k]) for k in ("pws", "rots", "scales", "shs", "alphas")}


def preprocess(g, cobj):
    return ops.surfel_preprocess_batch(g["pws"], g["rots"], g["scales"], g["shs"], g["alphas"], cobj)


def frame(W, H, pre, geo, capacity=False, records=None):
    """the batch frame on copies of us, depths, areas -> (outputs, depths and areas after the in-place culls)"""
    d, a = pre[1].clone(), pre[2].clone()
    f = ops.splat_surfel_geometry_batch if geo else ops.splat_surfel_batch
    return f(H, W, pre[0], d, a, pre[4] if records is None else records, capacity=capacity), d, a


def sc_of(s, cam):
    """scene s seen by one camera, as test_gpu_surfel_edges' scene dicts"""
    return dict(s, **cam)


# ---------------------------------------------------------------- the per-camera oracle
def camera_oracle(W, H, s, cam, pre, c, geo):
    """camera c's fp64 forward on the kernels' own records, binned by oracle.bin on the kernels' own u,
    depth and area -> dict(p (fp64 preprocess), rp (with the records' M, u, colour, n), bins, fwd)"""
    N = len(s["pws"])
    p = so.preprocess(s["pws"], s["rots"], s["scales"], s["shs"], cam["Rcw"], cam["tcw"], cam["twc"], cam["fx"],
                      cam["fy"], cam["cx"], cam["cy"])
    d, a = n(pre[1][c]).copy(), n(pre[2][c]).copy()
    bins = orc.bin(H, W, n(pre[0][c]), d, a) + (d, a)
    rp = record_pre(p, n(pre[4][c * N:(c + 1) * N]))
    fwd = (sgo.render_geometry if geo else so.render)(H, W, rp, s["alphas"], bins[:4])
    return dict(p=p, rp=rp, bins=bins, fwd=fwd)


def upstream(H, W, seed, geo):
    rng = np.random.default_rng(seed)
    return [rng.normal(size=sh) for sh in [(3, H, W), (H, W), (H, W), (3, H, W)] + [(H, W), (H, W)] * geo]


def oracle_rows(W, H, s, orac, dl, geo):
    """-> (rows, absolute sums) of the oracle's backward on dl (None: not given)"""
    if geo:
        return sgo.render_backward_geometry(H, W, orac["rp"], s["alphas"], orac["bins"][:4], orac["fwd"], *dl,
                                            abs_rows=True)
    return so.render_backward(H, W, orac["rp"], s["alphas"], orac["bins"][:4], orac["fwd"], *dl[:4], abs_rows=True)


def ratio(got, want, ab):
    """test_gpu_surfel_edges.rows_bound's ratio: |rows - oracle| / (1e-4 (the entry's absolute sum) + 1e-9
    max(absolute sums of its column))"""
    floor = 1e-9 * ab.max(axis=0, initial=0)[None, :] + 1e-30
    return np.abs(got.astype(np.float64) - want) / (1e-4 * ab + floor)


def check_rows(got, want, ab, kernel, scene):
    r = ratio(got, want, ab)
    key = (kernel, scene)
    WORST[key] = max(WORST.get(key, 0.0), float(r.max(initial=0)))
    assert r.max(initial=0) <= 1.0, (kernel, scene, float(r.max()), np.unravel_index(r.argmax(), r.shape))


def backward(W, H, pre, out, dl, geo, records=None):
    """the batch backward rasterizer on upstream planes dl ([C, ...] host arrays or None)"""
    td = [None if d is None else t(d) for d in dl]
    recs = pre[4] if records is None else records
    if geo:
        return ops.splatB_surfel_geometry_batch(H, W, recs, out[1], out[2], out[3], out[4], out[6], out[10], out[11],
                                                *td)
    return ops.splatB_surfel_batch(H, W, recs, out[1], out[2], out[3], out[4], *td[:4])


def rows_per_camera(W, H, s, cams, geo, label, masks=((1, 1, 1, 1, 1, 1),), records=None, sample=None, seed=0):
    """the batch frame and backward; camera c's rows (c in sample, default every camera) against its own
    oracle for every upstream subset in masks, the upstream planes zeroed on the oracle's ambiguous pixels.
    -> (pre, out, {c: oracle}, the full-mask upstream planes [C, ...], rows)"""
    C, N = len(cams), len(s["pws"])
    T = ((W + 15) // 16) * ((H + 15) // 16)
    cobj = gpu_cams(cams, W, H)
    pre = preprocess(gpu_scene(s), cobj)
    out, d, a = frame(W, H, pre, geo)
    sample = list(range(C)) if sample is None else sample
    orcs = {c: camera_oracle(W, H, s, cams[c], pre, c, geo) for c in sample}
    # camera c's tile lists: the oracle's on the kernels' own values
    ranges, gsid = n(out[3]), n(out[4])
    off = np.concatenate([[0], np.cumsum(np.diff(ranges, axis=1).reshape(C, T).sum(1))])
    for c, o in orcs.items():
        P, r, g = o["bins"][:3]
        assert off[c + 1] - off[c] == P, c
        assert np.array_equal(gsid[off[c]:off[c] + P] - c * N, g), c
        assert np.array_equal(np.where((r[:, 1] > r[:, 0])[:, None], r + off[c], 0), ranges[c * T:(c + 1) * T]), c
    kernel = "k_draw_2dgs_bwd_batch" if geo else "k_draw_disk_bwd_batch"
    ups = [upstream(H, W, seed + 100 * c, geo) for c in range(C)]
    for c, o in orcs.items():
        ok = ~o["fwd"]["ambiguous"]
        assert ok.mean() > 0.5, (c, ok.mean())
        ups[c] = [np.where(ok, d, 0.0).astype(np.float32) for d in ups[c]]
    full = [np.stack([u[i] for u in ups]) for i in range(len(ups[0]))]
    rows = None
    for mask in masks:
        dl = [d if m else None for d, m in zip(full, mask)]
        rows = backward(W, H, pre, out, dl, geo, records)
        got = n(rows)
        for c, o in orcs.items():
            want, ab = oracle_rows(W, H, s, o, [None if d is None else d[c] for d in dl], geo)
            check_rows(got[c * N:(c + 1) * N], want, ab, kernel, label)
    return pre, out, orcs, full, rows


# ---------------------------------------------------------------- (a) the backward rasterizers per entry
def odd_batch(C, W, H, N, k, seed):
    """N disks over camera 0's frame at 2-6 m, C cameras 0.03 rad and 0.1 m apart"""
    rng = np.random.default_rng(seed)
    cams = jittered_cameras(C, W, H, 0.8 * W, seed=seed, ang=0.03, shift=0.1)
    s = build(rng, [disks(rng, cams[0], W, H, N, (2.0, 6.0), margin=-4.0) + (rng.uniform(0.05, 0.95, N),)],
              cams[0], k)
    return cams, s


# upstream plane subsets (image, depth, alpha, normal, distortion, median); the disk kernel takes the first four
MASKS = ((1, 1, 1, 1, 1, 1), (0, 1, 0, 0, 1, 0), (1, 0, 1, 0, 0, 1), (0, 0, 0, 1, 0, 0))


@pytest.mark.parametrize("geo", [False, True], ids=["disk", "2dgs"])
@pytest.mark.parametrize("C", [2, 5])
def test_backward_rows_per_entry(C, geo):
    W, H = (53, 37) if C == 2 else (45, 29)
    cams, s = odd_batch(C, W, H, 250, 4, seed=C)
    masks = MASKS if C == 2 else MASKS[:1]
    rows_per_camera(W, H, s, cams, geo, "C%d %dx%d" % (C, W, H), masks=masks, seed=C)


@pytest.mark.parametrize("geo", [False, True], ids=["disk", "2dgs"])
def test_backward_rows_on_repacked_records(geo):
    """records re-packed from the C single-camera surfel_preprocess calls: their bits, and the rows per
    entry from them"""
    W, H, C = 45, 29, 3
    cams, s = odd_batch(C, W, H, 250, 9, seed=11)
    g = gpu_scene(s)
    cobj = gpu_cams(cams, W, H)
    single = [ops.surfel_preprocess(g["pws"], g["rots"], g["scales"], g["shs"], g["alphas"], c.Rcw, c.tcw, c.twc,
                                    c.fx, c.fy, c.cx, c.cy, W, H)[4] for c in cobj]
    recs = torch.cat(single)
    assert same(recs, preprocess(g, cobj)[4])
    rows_per_camera(W, H, s, cams, geo, "C3 re-packed", records=recs, seed=11)


@pytest.mark.parametrize("geo", [False, True], ids=["disk", "2dgs"])
def test_backward_rows_at_64_cameras(geo):
    C = ops.BATCH_MAX_CAMERAS
    W, H = 45, 29
    cams, s = odd_batch(C, W, H, 300, 16, seed=64)
    rng = np.random.default_rng(640 + geo)
    sample = [0, C - 1] + sorted(rng.choice(np.arange(1, C - 1), 4, replace=False).tolist())
    rows_per_camera(W, H, s, cams, geo, "C64", sample=sample, seed=64)


# ---------------------------------------------------------------- (b) the per-surfel batch kernels
def grads_reference(s, cams, rows, N, use=None):
    """the fp64 sum over cameras of so.preprocess_backward on each camera's rows, and each surfel's
    norm summed over cameras (test_gpu_surfel_batch.test_per_camera_against_the_oracles' bound);
    use [C,N]: the cameras each surfel's sum takes (default all)"""
    names = ("pws", "shs", "alphas", "scales", "rots")
    exp_sum, norm_sum = 0.0, 0.0
    for c, cam in enumerate(cams):
        p = so.preprocess(s["pws"], s["rots"], s["scales"], s["shs"], cam["Rcw"], cam["tcw"], cam["twc"], cam["fx"],
                          cam["fy"], cam["cx"], cam["cy"])
        r = rows[c * N:(c + 1) * N].astype(np.float64)
        ref = so.preprocess_backward(p, r)
        exp = np.concatenate([ref[k].reshape(N, -1) for k in names], 1)
        norm = np.maximum(np.linalg.norm(np.concatenate([exp, ref["us"]], 1), axis=1),
                          1e-3 * np.abs(p["K"]).sum() * np.linalg.norm(r, axis=1))
        if use is not None:
            exp, norm = np.where(use[c][:, None], exp, 0.0), np.where(use[c], norm, 0.0)
        exp_sum, norm_sum = exp_sum + exp, norm_sum + norm
    return exp_sum, norm_sum


def check_grads(g, s, cams, rows, N, what, use=None):
    """summed gradients against the fp64 sum (over the cameras in use); dL/dus[c] the rows' own entries"""
    got = np.concatenate([n(x).reshape(N, -1) for x in g[:5]], 1).astype(np.float64)
    assert np.isfinite(got).all() and np.isfinite(n(g[5])).all(), what
    exp, norm = grads_reference(s, cams, rows, N, use)
    err = np.abs(got - exp).max(axis=1)
    assert (err <= 1e-4 * norm + 1e-30).all(), (what, float((err / (norm + 1e-30)).max()))
    assert (n(g[3])[:, 2] == 0).all()
    for c in range(len(cams)):
        assert np.array_equal(n(g[5][c]), rows[c * N:(c + 1) * N, 16:18]), (what, c)


@pytest.mark.parametrize("k3", [1, 4, 9, 16])
def test_per_surfel_kernels_tails_and_alignment(k3):
    W, H, C = 64, 48, 3
    for N in (1, 127, 128, 129, 1000):
        rng = np.random.default_rng(10 * N + k3)
        cams = jittered_cameras(C, W, H, 0.8 * W, seed=N + k3, ang=0.03, shift=0.1)
        parts = disks(rng, cams[0], W, H, N, (2.0, 6.0), sigma=(1.0, 5.0))
        if N == 1:  # one disk at the frame's centre
            parts[0][0, :2] = [(W / 2 - cams[0]["cx"]) * parts[0][0, 2] / cams[0]["fx"], 0.0]
        s = build(rng, [parts + (rng.uniform(0.1, 0.95, N),)], cams[0], k3)
        g, cobj = gpu_scene(s), gpu_cams(cams, W, H)
        pre = preprocess(g, cobj)
        for c, cam in enumerate(cams):  # every camera's per-surfel outputs against the fp64 stages
            check_preprocess(sc_of(s, cam), g=[x[c] for x in pre[:4]] + [pre[4][c * N:(c + 1) * N]])
        out, _, _ = frame(W, H, pre, False)
        ups = [upstream(H, W, 7 * c + k3, False) for c in range(C)]
        rows = backward(W, H, pre, out, [np.stack([u[i] for u in ups]).astype(np.float32) for i in range(4)], False)
        rows_n = n(rows)
        for c in range(C):
            assert np.abs(rows_n[c * N:(c + 1) * N]).max() > 0, (N, c)
        gr = ops.surfel_preprocessB_batch(g["pws"], g["rots"], g["scales"], g["shs"], cobj, rows)
        check_grads(gr, s, cams, rows_n, N, (k3, N))
        for name in ("pws", "rots", "scales", "shs"):  # a view 4 bytes past a 16-byte boundary: the same bits
            g2 = dict(g, **{name: shifted(g[name])})
            pre2 = preprocess(g2, cobj)
            for x, y in zip(pre, pre2):
                assert same(x, y), (k3, N, name, "forward")
            gr2 = ops.surfel_preprocessB_batch(g2["pws"], g2["rots"], g2["scales"], g2["shs"], cobj, rows)
            for x, y in zip(gr, gr2):
                assert same(x, y), (k3, N, name, "backward")


# ---------------------------------------------------------------- (c) degenerate in one camera
def test_degenerate_in_one_camera():
    W, H, cams, s = special_batch()
    C, N = len(cams), len(s["pws"])
    pre, out, orcs, full, rows = rows_per_camera(W, H, s, cams, True, "special x7", seed=3)
    depths = n(pre[1])
    for c in range(C):  # the kernels cull exactly where the oracle does
        assert np.array_equal(depths[c] == -1, np.array(SPECIAL_KINDS[c]) == "culled"), c
    g = gpu_scene(s)
    gr = ops.surfel_preprocessB_batch(g["pws"], g["rots"], g["scales"], g["shs"], gpu_cams(cams, W, H), rows)
    rows_n = n(rows).reshape(C, N, -1)
    drawn = np.abs(rows_n).max(axis=2) > 0
    assert not drawn[depths == -1].any()
    assert not n(gr[5])[depths == -1].any()
    # every special surfel but the alpha-culled one is composited in some cameras and not in others
    for i in (0, 1, 2, 3, 4, 5, 6, 8, 9):
        assert drawn[:, i].any() and not drawn[:, i].all(), i
    assert not drawn[:, 7].any()
    check_grads(gr, s, cams, n(rows), N, "special", use=drawn)


# ---------------------------------------------------------------- (d) the tall frame's key plans
PLANS_REACHED = {}


@pytest.mark.parametrize("name", list(PLAN_BATCHES))
def test_tall_frame_key_plans(name):
    C, W, H, *_, want = PLAN_BATCHES[name]
    _, _, cams, s = plan_batch(name)
    N = len(s["pws"])
    T = ((W + 15) // 16) * ((H + 15) // 16)
    pre = preprocess(gpu_scene(s), gpu_cams(cams, W, H))
    bins = []
    for c in range(C):  # oracle.bin on the kernels' own u, depths and areas
        d, a = n(pre[1][c]).copy(), n(pre[2][c]).copy()
        bins.append(orc.bin(H, W, n(pre[0][c]), d, a) + (d, a))
    dk = depth_key_max(tall_keys(bins, T))
    p = key_plan(tall_height(C, H), W, dk)
    PLANS_REACHED[name] = ((p["tbits"], p["dbits"]), plan_shape(p))
    assert (p["tbits"],) + plan_shape(p) == (want[0],) + want[2:], (name, p)
    for geo in (False, True):
        exact, d, a = frame(W, H, pre, geo)
        check_cameras(exact, d, a, bins, N, T)
        frame(W, H, pre, geo, capacity=True)  # learns the bounds (the exact path)
        before = dict(ops.CAPACITY_STATS)
        cap, d2, a2 = frame(W, H, pre, geo, capacity=True)
        assert ops.CAPACITY_STATS["capacity_frames"] == before["capacity_frames"] + 1, "frame was redone"
        assert len(cap) == len(exact) == (12 if geo else 8)
        for i, (x, y) in enumerate(zip(exact, cap)):
            assert same(x, y), (name, geo, i)
        assert same(d, d2) and same(a, a2)
    print("tall plan %-10s (tbits, dbits) %s  %s" % (name, *PLANS_REACHED[name]))


# ---------------------------------------------------------------- (e) frame boundaries
def test_frame_boundaries_in_the_geometry_backward():
    C, W, H = BOUNDARY
    _, _, cams, s, edge = boundary_batch()
    N = len(s["pws"])
    pre, out, orcs, full, rows = rows_per_camera(W, H, s, cams, True, "boundary C3 70x45", seed=45)
    rows_n = n(rows)
    alpha = n(out[6])
    for c in range(C):  # the edge disks are drawn on frame c's last and first rows
        bottom, top = edge[c]
        xs = lambda ids: np.round(n(pre[0][c])[ids, 0]).astype(int)
        assert (alpha[c, H - 1, xs(bottom)] > 0.1).all() and (alpha[c, 0, xs(top)] > 0.1).all(), c
        assert (np.abs(rows_n[c * N + bottom]).max(axis=1) > 0).all()
    for c in range(C):
        # frame c's upstream planes alone: camera c's rows as in the full run (float atomics: within the
        # per-entry bound), every other camera's rows exactly 0
        dl = [np.where((np.arange(C) == c).reshape((C,) + (1,) * (d.ndim - 1)), d, 0).astype(np.float32)
              for d in full]
        one = n(backward(W, H, pre, out, dl, True))
        _, ab = oracle_rows(W, H, s, orcs[c], [d[c] for d in dl], True)
        check_rows(one[c * N:(c + 1) * N], rows_n[c * N:(c + 1) * N].astype(np.float64), ab,
                   "k_draw_2dgs_bwd_batch", "frame %d alone" % c)
        others = np.ones(C * N, bool)
        others[c * N:(c + 1) * N] = False
        assert not one[others].any(), c
