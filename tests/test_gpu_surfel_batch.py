"""Batched 2D Gaussian Splatting (DESIGN 3.25) on the GPU.

1. Forward: camera c's per-surfel outputs, planes (colour and geometry frames) and tile lists from the
   batch are the bits of the single-camera calls, at C in {1, 3, 8} and every SH degree.
2. Per camera against the fp64 oracles (oracle/surfel_oracle.py, tests/surfel_geometry_oracle.py), which
   never see a batch: the planes and the 18-float gradient rows.
3. Backward: rows, summed per-surfel gradients and dL/dus[c] against the C single-camera calls (1e-5 of
   each tensor's max |g|: the rasterizer backward sums rows with float atomics); upstream plane subsets;
   no backward rasterizer when no plane has a gradient.
4. Tall-frame edges: a surfel across frame c's bottom edge, the 2^24 area cap in one camera, a camera
   that sees nothing, whole-tile entries, N = 0, C = 64, C gy = 65535 tile rows accepted and one more
   refused, the capacity path against the exact one and an outgrown capacity redone.
5. A short 2DGS training run with C = 4 views per step against the loop of single calls."""
import numpy as np
import pytest
import torch

from oracle import surfel_oracle as so
import surfel_geometry_oracle as sgo
from test_surfel_edge_scenes_cpu import camera, special_scene

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def n(t):
    return t.detach().cpu().numpy()


def ops():
    from easygaussiansplatting_b200 import ops as o
    return o


def scene(N, W, H, k=16, seed=0, z=(2.0, 6.0), spread=1.0):
    rng = np.random.default_rng(seed)
    f = 0.8 * W
    zz = rng.uniform(*z, N)
    pws = np.stack([rng.uniform(-spread, spread, N) * zz * W / (2 * f), rng.uniform(-spread, spread, N) * zz * H / (2 * f),
                    zz], 1)
    scales = np.stack([rng.uniform(0.02, 0.15, N), rng.uniform(0.02, 0.15, N), rng.uniform(0.0, 0.05, N)], 1)
    f32 = lambda a: T(np.asarray(a, dtype=np.float32))
    return dict(pws=f32(pws), rots=f32(rng.normal(size=(N, 4))), scales=f32(scales),
                shs=f32(rng.normal(scale=0.3, size=(N, 3 * k))), alphas=f32(rng.uniform(0.05, 0.95, N)))


def cameras(C, W, H, seed=0, poses=None):
    """C pinhole cameras of one size: small rotations and offsets around the origin, intrinsics of their own"""
    from easygaussiansplatting_b200.gsfunction import Camera
    rng = np.random.default_rng(seed + 1000)
    cams = []
    for c in range(C):
        if poses is not None:
            Rcw, tcw, twc = poses[c]
        else:
            a = rng.normal(size=3) * 0.05
            K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
            Rcw = np.eye(3) + np.sin(np.linalg.norm(a)) / max(np.linalg.norm(a), 1e-12) * K + \
                (1 - np.cos(np.linalg.norm(a))) / max(np.linalg.norm(a), 1e-12) ** 2 * K @ K
            twc = rng.normal(size=3) * 0.1
            tcw = -Rcw @ twc
        f = 0.8 * W * (1 + 0.03 * rng.normal())
        cams.append(Camera(W, H, f, f * (1 + 0.01 * c), W / 2 - 0.3 + 0.2 * rng.normal(), H / 2 + 0.2 + 0.2 * rng.normal(),
                           T(np.float32(Rcw)), T(np.float32(tcw)), T(np.float32(twc))))
    return cams


def single_pre(s, cam):
    return ops().surfel_preprocess(s["pws"], s["rots"], s["scales"], s["shs"], s["alphas"], cam.Rcw, cam.tcw, cam.twc,
                                   cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height)


def single_frame(s, cam, geo, capacity=False):
    pre = single_pre(s, cam)
    us, depths, areas, _, recs = pre
    if geo:
        out = ops().splat_surfel_geometry(cam.height, cam.width, us, depths, areas, recs, capacity=capacity)
    else:
        out = ops().splat_surfel(cam.height, cam.width, us, depths, areas, recs, capacity=capacity)
    return pre, out


def batch_frame(s, cams, geo, capacity=False):
    o = ops()
    pre = o.surfel_preprocess_batch(s["pws"], s["rots"], s["scales"], s["shs"], s["alphas"], cams)
    raw = [t.clone() for t in pre]  # (the binning culls depths / areas in place)
    us, depths, areas, _, recs = pre
    H, W = cams[0].height, cams[0].width
    if geo:
        out = o.splat_surfel_geometry_batch(H, W, us, depths, areas, recs, capacity=capacity)
    else:
        out = o.splat_surfel_batch(H, W, us, depths, areas, recs, capacity=capacity)
    return raw, pre, out


def tile_lists(ranges, gsid):
    r, g = n(ranges), n(gsid)
    return [g[a:b] for a, b in r]


def assert_frames_equal(s, cams, geo, capacity=False, batch=None):
    """frame c of the batch == the single frame of camera c, every plane and the tile lists with ids
    c N + n -> n; no tile of frame c lists a record of another camera"""
    N = s["pws"].shape[0]
    raw, pre, out = batch_frame(s, cams, geo, capacity) if batch is None else batch
    H, W = cams[0].height, cams[0].width
    Tn = ((W + 15) // 16) * ((H + 15) // 16)
    lists = tile_lists(out[3], out[4])
    for c, cam in enumerate(cams):
        spre = [t.clone() for t in single_pre(s, cam)]
        for i, (a, b) in enumerate(zip(raw, spre)):
            a = a[c * N:(c + 1) * N] if i == 4 else a[c]
            assert torch.equal(a, b), ("per-surfel output", i, c)
        _, sout = single_frame(s, cam, geo)
        for i in [0, 1, 2] + list(range(5, len(out))):
            assert torch.equal(out[i][c], sout[i]), ("plane", i, c)
        slists = tile_lists(sout[3], sout[4])
        for t in range(Tn):
            got = lists[c * Tn + t]
            assert ((got // max(N, 1)) == c).all(), ("foreign record in frame", c, t)
            assert np.array_equal(got - c * N, slists[t]), ("tile list", c, t)
    return raw, pre, out


# ---------------------------------------------------------------- 1. forward bits
@pytest.mark.parametrize("k", [1, 4, 9, 16])
@pytest.mark.parametrize("C", [1, 3, 8])
def test_forward_bits_match_single_calls(C, k):
    W, H = 83, 61  # partial tiles in both directions
    s = scene(1500, W, H, k=k, seed=C * 10 + k, spread=1.2)
    cams = cameras(C, W, H, seed=C + k)
    for geo in (False, True):
        raw, _, out = assert_frames_equal(s, cams, geo)
        assert n(out[4]).size > 0
        lens = np.diff(n(out[3]), axis=1)
        assert lens.max() > 32  # per-block entries as well as whole-tile ones


# ---------------------------------------------------------------- 2. per camera against the oracles
def upstream(C, H, W, seed=1, geo=False):
    rng = np.random.default_rng(seed)
    shapes = [(C, 3, H, W), (C, H, W), (C, H, W), (C, 3, H, W)] + ([(C, H, W), (C, H, W)] if geo else [])
    return [rng.normal(size=sh).astype(np.float32) for sh in shapes]


def test_per_camera_against_the_oracles():
    o = ops()
    W, H, C = 72, 48, 3
    s = scene(600, W, H, k=9, seed=21, spread=1.1)
    cams = cameras(C, W, H, seed=5)
    raw, pre, out = batch_frame(s, cams, True)
    N = s["pws"].shape[0]
    npre = {k: n(v) for k, v in s.items()}
    dls, oracle = [], []
    for c, cam in enumerate(cams):
        p = so.preprocess(npre["pws"], npre["rots"], npre["scales"], npre["shs"], n(cam.Rcw), n(cam.tcw), n(cam.twc),
                          cam.fx, cam.fy, cam.cx, cam.cy)
        bins = so.orc.bin(H, W, n(pre[0][c]), n(raw[1][c]).copy(), n(raw[2][c]).copy())
        fwd = sgo.render_geometry(H, W, p, npre["alphas"], bins)
        ok = ~fwd["ambiguous"]
        assert ok.mean() > 0.95
        for i, name in ((0, "image"), (7, "normal")):
            assert np.abs(n(out[i][c]) - fwd[name]).max(axis=0)[ok].max() < 1e-4, (name, c)
        assert np.abs(n(out[6][c]) - fwd["alpha"])[ok].max() < 1e-4
        assert np.abs(n(out[5][c]) - fwd["depth"])[ok].max() < 1e-4 * max(1.0, np.abs(fwd["depth"]).max())
        assert np.abs(n(out[8][c]) - fwd["distortion"])[ok].max() < 1e-4 * max(1.0, np.abs(fwd["distortion"]).max())
        assert np.abs(n(out[9][c]) - fwd["median_depth"])[ok].max() < 1e-4 * max(1.0, fwd["median_depth"].max())
        assert (n(out[1][c]) == fwd["contrib"])[ok].all()
        # the rows against the oracle run on the kernels' own records (M, u, colour, n of camera c), as
        # test_gpu_surfel_edges compares them: the rasterizers on their own inputs
        r = n(pre[4][c * N:(c + 1) * N]).astype(np.float64)
        rp = dict(p, M=r[:, :9].reshape(-1, 3, 3), u=r[:, 10:12], colors=r[:, 14:17], n=r[:, 17:20])
        fwd_r = sgo.render_geometry(H, W, rp, npre["alphas"], bins)
        amb = fwd["ambiguous"] | fwd_r["ambiguous"]
        dl = [np.where(amb, 0.0, d[c]).astype(np.float32) for d in upstream(C, H, W, seed=c, geo=True)]
        dls.append(dl)
        oracle.append((p, *sgo.render_backward_geometry(H, W, rp, npre["alphas"], bins, fwd_r, *dl, abs_rows=True)))
    dl = [T(np.stack([d[i] for d in dls])) for i in range(6)]
    rows = o.splatB_surfel_geometry_batch(H, W, pre[4], out[1], out[2], out[3], out[4], out[6], out[10], out[11],
                                          *dl)
    g = o.surfel_preprocessB_batch(s["pws"], s["rots"], s["scales"], s["shs"], cams, rows)
    names = ("pws", "shs", "alphas", "scales", "rots")
    exp_sum, norm_sum = 0.0, 0.0
    for c, (p, want, ab) in enumerate(oracle):
        # test_gpu_surfel_edges' two stages: the rows per entry within 1e-4 of the entry's sum of absolute
        # per-pixel terms, then the per-surfel pass on the kernels' own rows relative to each surfel's norm
        got = n(rows[c * N:(c + 1) * N]).astype(np.float64)
        floor = 1e-9 * ab.max(axis=0, initial=0)[None, :] + 1e-30
        assert (np.abs(got - want) / (1e-4 * ab + floor)).max(initial=0) <= 1.0, c
        ref = so.preprocess_backward(p, got)
        exp = np.concatenate([ref[k].reshape(N, -1) for k in names], 1)
        norm = np.maximum(np.linalg.norm(np.concatenate([exp, ref["us"]], 1), axis=1),
                          1e-3 * np.abs(p["K"]).sum() * np.linalg.norm(got, axis=1))
        assert (np.abs(n(g[5][c]) - ref["us"]).max(axis=1) <= 1e-4 * norm + 1e-30).all(), c
        exp_sum, norm_sum = exp_sum + exp, norm_sum + norm
    got = np.concatenate([n(x).reshape(N, -1) for x in g[:5]], 1).astype(np.float64)
    assert (np.abs(got - exp_sum).max(axis=1) <= 1e-4 * norm_sum + 1e-30).all()


# ---------------------------------------------------------------- 3. backward against the single calls
def close(a, b, what, tol=1e-5):
    a, b = n(a), n(b)
    assert a.shape == b.shape, what
    assert np.abs(a - b).max() <= tol * max(np.abs(b).max(), 1e-30), what


def single_grads(s, cam, out, dl, geo):
    o = ops()
    pre = single_pre(s, cam)
    if geo:
        rows = o.splatB_surfel_geometry(cam.height, cam.width, pre[4], out[1], out[2], out[3], out[4], out[6], out[10],
                                        out[11], *dl)
    else:
        rows = o.splatB_surfel(cam.height, cam.width, pre[4], out[1], out[2], out[3], out[4], *dl[:4])
    g = o.surfel_preprocessB(s["pws"], s["rots"], s["scales"], s["shs"], cam.Rcw, cam.tcw, cam.twc, cam.fx, cam.fy,
                             cam.cx, cam.cy, cam.width, cam.height, rows)
    return rows, g


@pytest.mark.parametrize("geo", [False, True], ids=["surfel", "geometry"])
@pytest.mark.parametrize("mask", [(1, 1, 1, 1, 1, 1), (0, 1, 0, 0, 1, 0), (0, 0, 0, 1, 0, 1), (1, 0, 1, 0, 0, 0)])
def test_backward_is_the_sum_of_single_calls(geo, mask):
    o = ops()
    W, H, C = 90, 60, 3
    s = scene(2000, W, H, k=16, seed=31, spread=1.1)
    cams = cameras(C, W, H, seed=7)
    _, pre, out = batch_frame(s, cams, geo)
    N = s["pws"].shape[0]
    dl = [T(d) if m else None for d, m in zip(upstream(C, H, W, seed=2, geo=True), mask)]
    if geo:
        rows = o.splatB_surfel_geometry_batch(H, W, pre[4], out[1], out[2], out[3], out[4], out[6], out[10], out[11],
                                              *dl)
    else:
        rows = o.splatB_surfel_batch(H, W, pre[4], out[1], out[2], out[3], out[4], *dl[:4])
    g = o.surfel_preprocessB_batch(s["pws"], s["rots"], s["scales"], s["shs"], cams, rows)
    total = None
    for c, cam in enumerate(cams):
        _, sout = single_frame(s, cam, geo)
        srows, sg = single_grads(s, cam, sout, [None if d is None else d[c] for d in dl], geo)
        close(rows[c * N:(c + 1) * N], srows, ("rows", c))
        close(g[5][c], sg[5], ("dus", c))
        total = list(sg[:5]) if total is None else [a + b for a, b in zip(total, sg[:5])]
    for i, name in enumerate(("pws", "shs", "alphas", "scales", "rots")):
        close(g[i], total[i], name)
    assert (n(g[3])[:, 2] == 0).all()


@pytest.mark.parametrize("geo", [False, True], ids=["surfel", "geometry"])
def test_autograd_and_no_backward_rasterizer_without_a_plane_gradient(geo):
    from easygaussiansplatting_b200 import _lib
    from easygaussiansplatting_b200.gsfunction import GSFunctionSurfelBatch, GSFunctionSurfelGeometryBatch
    W, H, C = 64, 40, 3
    s = scene(400, W, H, k=4, seed=41)
    cams = cameras(C, W, H, seed=9)
    P = {k: s[k].clone().requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    al = s["alphas"][:, None].clone().requires_grad_()
    us = torch.zeros((C, 400, 2), device=DEV, requires_grad=True)
    fn = GSFunctionSurfelGeometryBatch if geo else GSFunctionSurfelBatch
    outs = fn.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us, cams)
    assert len(outs) == (7 if geo else 5) and outs[-1].shape == (C, 400) and outs[-1].dtype == torch.bool
    dl = [T(d) for d in upstream(C, H, W, seed=3, geo=geo)]
    sum((p * d).sum() for p, d in zip(outs[:-1], dl)).backward()
    _, pre, out = batch_frame(s, cams, geo)
    for i, o_ in enumerate(outs[:-1]):
        ref = out[[0, 5, 6, 7, 8, 9][i]]
        assert torch.equal(o_.detach(), ref), i
    total = None
    for c, cam in enumerate(cams):
        _, sout = single_frame(s, cam, geo)
        _, sg = single_grads(s, cam, sout, [d[c] for d in dl] + [None, None] * (not geo), geo)
        close(us.grad[c], sg[5], ("us", c))
        total = list(sg[:5]) if total is None else [a + b for a, b in zip(total, sg[:5])]
    for name, t, i in (("pws", P["pws"], 0), ("shs", P["shs"], 1), ("scales", P["scales"], 3), ("rots", P["rots"], 4)):
        close(t.grad, total[i], name)
    close(al.grad[:, 0], total[2], "alphas")
    # one plane with a gradient: one launch of the plain batched backward rasterizer; none: no launch
    lib = _lib.load()
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    kids = [names.index(k) for k in ("draw_surfel_backward_batch", "draw_2dgs_backward_batch")]
    n0 = [lib.gsb_profile_launches(k) for k in kids]
    outs = fn.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us, cams)
    (outs[2].sum() * 0).backward()
    torch.cuda.synchronize()
    assert [lib.gsb_profile_launches(k) for k in kids] == [n0[0] + 1, n0[1]]
    rows = ops().splatB_surfel_batch(H, W, pre[4], out[1], out[2], out[3], out[4])
    torch.cuda.synchronize()
    assert [lib.gsb_profile_launches(k) for k in kids] == [n0[0] + 1, n0[1]] and not n(rows).any()


def test_refusals():
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionSurfelBatch, GSFunctionSurfelGeometryBatch
    W, H = 32, 24
    s = scene(10, W, H, k=1)
    cams = cameras(2, W, H)
    us = torch.zeros((2, 10, 2), device=DEV)
    a = (s["pws"], s["shs"], s["alphas"][:, None], s["scales"], s["rots"], us)
    e = torch.eye(3, device=DEV)
    z = torch.zeros(3, device=DEV)
    bad = [Camera(W, H, 20, 20, 16, 12, e, z, antialiased=True),
           Camera(W, H, 20, 20, 16, 12, e, z, camera_model="ortho"),
           Camera(W + 16, H, 20, 20, 16, 12, e, z)]
    for fn in (GSFunctionSurfelBatch, GSFunctionSurfelGeometryBatch):
        for b in bad:
            with pytest.raises(ValueError):
                fn.apply(*a, [cams[0], b])
        ge = cameras(2, W, H)
        ge[1].grad_exchange = object()
        with pytest.raises(ValueError):
            fn.apply(*a, ge)
        with pytest.raises(ValueError):
            fn.apply(*a[:5], torch.zeros((3, 10, 2), device=DEV), cams)
    with pytest.raises(ValueError):
        GSFunctionSurfelBatch.apply(*a, cams, torch.zeros(10, device=DEV))
    with pytest.raises(ValueError):
        GSFunctionSurfelBatch.apply(*a, cams, None, torch.zeros((2, 10, 2), device=DEV))
    with pytest.raises(ValueError):
        GSFunctionSurfelGeometryBatch.apply(*a, cams, torch.zeros(1, device=DEV))


# ---------------------------------------------------------------- 4. tall-frame edges
def test_bottom_edge_grazing_cap_blind_camera_and_whole_tiles():
    """camera posed_b sees the special scene's surfel 8 at the 2^24 area cap; one camera looks away
    (sees nothing); a surfel straddles the bottom edge of every frame; a sparse scene has whole-tile
    entries only"""
    sc = special_scene(k=4, cam="posed_b")
    W, H = sc["W"], sc["H"]
    s = {k: T(sc[k]) for k in ("pws", "rots", "scales", "shs", "alphas")}
    # a surfel centred one pixel above the bottom edge of posed_b's frame, 6 px across
    Rcw, tcw, _ = camera("posed_b")
    f = sc["fx"]
    pc = np.array([(40.0 - sc["cx"]) * 3.0 / f, (H - 1.0 - sc["cy"]) * 3.0 / f, 3.0])
    s["pws"] = torch.cat([s["pws"], T(np.float32((pc - tcw) @ Rcw))[None]])
    s["rots"] = torch.cat([s["rots"], T(np.float32([1, 0, 0, 0]))[None]])
    s["scales"] = torch.cat([s["scales"], T(np.float32([0.08, 0.08, 0]))[None]])
    s["shs"] = torch.cat([s["shs"], s["shs"][:1]])
    s["alphas"] = torch.cat([s["alphas"], T(np.float32([0.9]))])
    Rb, _, twb = camera("posed_b")
    Ra = np.diag([-1.0, 1.0, -1.0]) @ Rb  # posed_b turned around: every surfel behind it
    away = (Ra, -Ra @ twb, twb)
    poses = [camera("identity"), camera("posed_b"), away, camera("posed_b")]
    from easygaussiansplatting_b200.gsfunction import Camera
    cams = [Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(np.float32(R)), T(np.float32(t)), T(np.float32(tw)))
            for R, t, tw in poses]
    N = s["pws"].shape[0]
    for geo in (False, True):
        raw, pre, out = assert_frames_equal(s, cams, geo)
        assert (n(raw[2][1][8]) == so.AREA_CAP).any() and n(raw[1][1][8]) > 0
        assert (n(raw[1][2]) == -1).all() and not n(out[0][2]).any() and not n(out[6][2]).any()
        # the edge surfel is drawn on frame 1's last row and not carried into frame 2's first tile row
        assert n(out[6][1])[H - 1, 36:45].max() > 0.1
        Tn = ((W + 15) // 16) * ((H + 15) // 16)
        assert (n(out[4]) == N + N - 1).any()
        r = n(out[3])[2 * Tn:3 * Tn]
        assert (r[:, 1] == r[:, 0]).all()
    # whole-tile entries only
    s2 = scene(40, 80, 48, k=1, seed=51)
    raw, pre, out = assert_frames_equal(s2, cameras(3, 80, 48, seed=51), False)
    lens = np.diff(n(out[3]), axis=1)
    assert 0 < lens.max() <= 32


def test_empty_batch():
    from easygaussiansplatting_b200.gsfunction import GSFunctionSurfelGeometryBatch
    W, H, C = 33, 17, 2
    s = scene(0, W, H, k=1)
    cams = cameras(C, W, H)
    for geo in (False, True):
        raw, pre, out = assert_frames_equal(s, cams, geo)
        assert all(not n(t).any() for t in out[:3] + out[5:])
    P = {k: s[k].clone().requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    al = s["alphas"][:, None].clone().requires_grad_()
    us = torch.zeros((C, 0, 2), device=DEV, requires_grad=True)
    outs = GSFunctionSurfelGeometryBatch.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us, cams)
    sum(o.sum() for o in outs[:6]).backward()
    assert P["pws"].grad.shape == (0, 3) and us.grad.shape == (C, 0, 2)


def test_64_cameras():
    o = ops()
    C = o.BATCH_MAX_CAMERAS
    W, H = 45, 29
    s = scene(300, W, H, k=16, seed=64)
    cams = cameras(C, W, H, seed=64)
    raw, pre, out = assert_frames_equal(s, cams, True)
    N = 300
    dl = [T(d) for d in upstream(C, H, W, seed=6, geo=True)]
    rows = o.splatB_surfel_geometry_batch(H, W, pre[4], out[1], out[2], out[3], out[4], out[6], out[10], out[11], *dl)
    g = o.surfel_preprocessB_batch(s["pws"], s["rots"], s["scales"], s["shs"], cams, rows)
    total = None
    for c, cam in enumerate(cams):
        _, sout = single_frame(s, cam, True)
        srows, sg = single_grads(s, cam, sout, [d[c] for d in dl], True)
        close(rows[c * N:(c + 1) * N], srows, ("rows", c))
        close(g[5][c], sg[5], ("dus", c))
        total = list(sg[:5]) if total is None else [a + b for a, b in zip(total, sg[:5])]
    for i in range(5):
        close(g[i], total[i], i)
    with pytest.raises(ValueError):
        o.surfel_preprocess_batch(s["pws"], s["rots"], s["scales"], s["shs"], s["alphas"], cams + cams[:1])


def test_tall_frame_row_limit():
    """3 frames of 21845 tile rows (65535 in all) are drawn; 21846 rows each are refused before any launch"""
    o = ops()
    free, _ = torch.cuda.mem_get_info()
    if free < (4 << 30):
        pytest.skip("needs 4 GiB of free device memory")
    W, H, C = 32, 16 * 21845, 3
    rng = np.random.default_rng(77)
    N = 60
    f = 40.0
    # surfels on the first and last tile rows of every frame and a few in between
    v = np.concatenate([rng.uniform(0, 30, N // 3), rng.uniform(H - 30, H, N // 3), rng.uniform(0, H, N - 2 * (N // 3))])
    uu = rng.uniform(0, W, N)
    z = rng.uniform(2, 4, N)
    cy = H / 2
    pws = np.stack([(uu - 16) * z / f, (v - cy) * z / f, z], 1)
    s = dict(pws=T(np.float32(pws)), rots=T(np.float32(rng.normal(size=(N, 4)))),
             scales=T(np.float32(np.stack([rng.uniform(0.05, 0.2, N), rng.uniform(0.05, 0.2, N), np.zeros(N)], 1))),
             shs=T(np.float32(rng.normal(scale=0.3, size=(N, 3)))), alphas=T(np.float32(rng.uniform(0.2, 0.9, N))))
    from easygaussiansplatting_b200.gsfunction import Camera
    e, z3 = np.eye(3, dtype=np.float32), np.zeros(3, np.float32)
    cams = [Camera(W, H, f, f, 16 + 0.1 * c, cy + 0.1 * c, T(e), T(z3), T(z3)) for c in range(C)]
    pre = o.surfel_preprocess_batch(s["pws"], s["rots"], s["scales"], s["shs"], s["alphas"], cams)
    out = o.splat_surfel_batch(H, W, *pre[:3], pre[4])
    for c in (0, C - 1):
        _, sout = single_frame(s, cams[c], False)
        for i in (0, 1, 2, 5, 6, 7):
            assert torch.equal(out[i][c], sout[i]), (c, i)
        assert n(out[6][c])[:16].any() and n(out[6][c])[-16:].any()
    del out
    cams2 = [Camera(W, H + 16, f, f, 16, cy, T(e), T(z3), T(z3)) for _ in range(C)]
    pre = o.surfel_preprocess_batch(s["pws"], s["rots"], s["scales"], s["shs"], s["alphas"], cams2)
    with pytest.raises(RuntimeError, match="65535"):
        o.splat_surfel_batch(H + 16, W, *pre[:3], pre[4])


def test_capacity_path_matches_exact_path():
    o = ops()
    W, H, C = 96, 64, 4
    s = scene(5000, W, H, k=16, seed=91)
    cams = cameras(C, W, H, seed=91)
    for geo in (False, True):
        exact = batch_frame(s, cams, geo)
        stats = dict(o.CAPACITY_STATS)
        batch_frame(s, cams, geo, capacity=True)          # exact, learns the bounds
        second = batch_frame(s, cams, geo, capacity=True)  # the capacity path
        assert o.CAPACITY_STATS["capacity_frames"] > stats["capacity_frames"]
        for a, b in zip(exact[2], second[2]):
            assert torch.equal(a, b)
        assert_frames_equal(s, cams, geo, batch=second)
        big = dict(s)
        big["scales"] = s["scales"] * 2.5
        outgrown = o.CAPACITY_STATS["outgrown"]
        got = batch_frame(big, cams, geo, capacity=True)
        assert o.CAPACITY_STATS["outgrown"] == outgrown + 1
        ref = batch_frame(big, cams, geo)
        for a, b in zip(got[2], ref[2]):
            assert torch.equal(a, b)


# ---------------------------------------------------------------- 5. training
def test_training_with_four_views_per_step():
    """2DGS with the geometry terms, C = 4 views per step, per-camera DensityController statistics and
    GaussianAdam: the batch lowers the loss as the loop of single calls does, and their losses agree"""
    from easygaussiansplatting_b200.density import DensityController
    from easygaussiansplatting_b200.gsfunction import GSFunctionSurfelGeometry, GSFunctionSurfelGeometryBatch
    from easygaussiansplatting_b200.loss import depth_to_normal
    from easygaussiansplatting_b200.optim import GaussianAdam
    W, H, C, N = 64, 48, 4, 1500
    cams = cameras(C, W, H, seed=111)
    gt_scene = scene(N, W, H, k=4, seed=112)
    with torch.no_grad():
        us0 = torch.zeros((C, N, 2), device=DEV)
        gt = GSFunctionSurfelGeometryBatch.apply(gt_scene["pws"], gt_scene["shs"], gt_scene["alphas"][:, None],
                                                 gt_scene["scales"], gt_scene["rots"], us0, cams)[0]
    start = scene(N, W, H, k=4, seed=113)

    def run(batch, steps=25):
        P = {k: start[k].clone().requires_grad_() for k in ("pws", "shs", "scales", "rots")}
        P["alphas"] = start["alphas"][:, None].clone().requires_grad_()
        opt = GaussianAdam([{"params": [P[k]], "name": k, "lr": lr} for k, lr in
                            (("pws", 2e-3), ("shs", 2e-2), ("scales", 2e-3), ("rots", 2e-3), ("alphas", 2e-2))])
        dc = DensityController(1.0, verbose=False)
        losses = []
        for _ in range(steps):
            opt.zero_grad()
            a = (P["pws"], P["shs"], P["alphas"], P["scales"], P["rots"])
            if batch:
                us = torch.zeros((C, N, 2), device=DEV, requires_grad=True)
                image, depth, alpha, normal, dist, med, mask = GSFunctionSurfelGeometryBatch.apply(*a, us, cams)
                nd = depth_to_normal(med, cams)
                ln = (1 - (normal * nd * alpha.detach()[:, None]).sum(1)).mean()
                loss = (image - gt).abs().mean() + 0.1 * dist.mean() + 0.01 * ln
                loss.backward()
                for c in range(C):
                    dc.update_density_info(us.grad[c], mask[c])
            else:
                loss, uss, masks = 0.0, [], []
                for c, cam in enumerate(cams):
                    us = torch.zeros((N, 2), device=DEV, requires_grad=True)
                    image, depth, alpha, normal, dist, med, mask = GSFunctionSurfelGeometry.apply(*a, us, cam)
                    ln = (1 - (normal * depth_to_normal(med, cam) * alpha.detach()).sum(0)).mean()
                    loss = loss + ((image - gt[c]).abs().mean() + 0.1 * dist.mean() + 0.01 * ln) / C
                    uss.append(us); masks.append(mask)
                loss.backward()
                for us, mask in zip(uss, masks):
                    dc.update_density_info(us.grad, mask)
            opt.step()
            losses.append(float(loss.detach()))
        return losses, dc

    lb, dcb = run(True)
    ll, dcl = run(False)
    assert lb[-1] < 0.8 * lb[0] and ll[-1] < 0.8 * ll[0]
    assert abs(lb[0] - ll[0]) <= 1e-5 * ll[0]
    assert abs(lb[-1] - ll[-1]) <= 2e-2 * ll[-1]
    assert torch.equal(dcb.cunt, dcl.cunt)
    close(dcb.grad_accum, dcl.grad_accum, "grad_accum", tol=1e-2)
