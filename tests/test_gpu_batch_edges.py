"""Batched rendering (DESIGN 3.21) at the edges of its tall frame, against independent oracles.

(a) every key plan the tall frame can pick -- one to four passes of 9- or 8-bit digits, key widths of 32
    and 33 bits, full and saturated depth keys in the 64-bit layout, and two batches whose every single
    frame sorts 32-bit keys while the tall frame needs the 64-bit layout (one of them only because of a
    far Gaussian seen by one camera) -- bit for bit against `oracle.bin` per camera, exact and capacity path;
(b) the tall frame at the 65535-tile-row limit (3 x 21845 rows) and at C = 64 (64 x 1023 rows), with
    Gaussians on the first and last rows of every camera, straddling every camera boundary and far past
    it: tile lists and planes per camera against `oracle.splat`, the first and last cameras also bit for
    bit against the single-camera `ops.splat`;
(c) the batch capacity path with the learnt patch bound at P and P - 1 and a batch whose depth keys
    outgrow the learnt plan, in the narrow and the 64-bit layout, colour and RGB-D;
(d) k_draw_bwd_batch and k_draw_bwd_rgbd_batch per entry against each camera's own fp64 conditioning
    (test_gpu_raster_rows' bounds), with a different scene in every camera and pad rows in every frame;
(e) orthographic, fisheye and OpenCV batches through GSFunctionFusedBatch[RGBD] against the fp64
    whole-step oracles, at the single-camera whole-step tests' bounds;
(f) C = 64 against the loop of single-camera calls, and per entry for the first and the last camera.

The scene builders of (a) - (c) are in test_batch_edges_cpu.py, which checks that each reaches its plan."""
import numpy as np
import pytest
import torch

from oracle import absgrad_oracle as oabs
from oracle import camera_model_oracle as ocm
from oracle import opencv_oracle as ocv
from oracle import oracle as orc
from oracle import rgbd_oracle as orgbd
from easygaussiansplatting_b200 import ops
from easygaussiansplatting_b200.gsfunction import (Camera, GSFunctionFused, GSFunctionFusedBatch,
                                                   GSFunctionFusedBatchRGBD)
from easygaussiansplatting_b200.scene import (COLMAP_LIKE_FISHEYE_K, COLMAP_LIKE_OPENCV, camera_model_scene,
                                              upstream_gradient)

from test_batch_edges_cpu import (BATCH_PLANS, ROW_LIMIT, batch_plan_scene, camera_bins, capacity_scene, key_plan,
                                  plan_shape, row_limit_scene, tall_height, tall_keys)
from test_gpu_batch import _cams as batch_cams
from test_gpu_batch import _close as close_max
from test_gpu_batch import _params as batch_params
from test_gpu_binning import need_free_memory, widths
from test_gpu_camera_model import _close as close_rows
from test_gpu_raster_rows import WORST, check, check_flagged, check_moments, scene_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def fresh_capacities():
    ops._CAPACITY.clear()
    yield
    ops._CAPACITY.clear()


@pytest.fixture(scope="module", autouse=True)
def report_worst_ratios():
    yield
    for (kernel, scene), r in sorted(WORST.items()):
        if kernel.endswith("_batch"):
            print("worst ratio %-22s %-36s %.3e" % (kernel, scene, r))


def t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).to(DEV)


def n(x):
    return x.detach().cpu().numpy()


def same(x, y):
    return torch.equal(x.view(torch.int32), y.view(torch.int32))


def fillers(C, N, seed):
    """conics, opacities and colours of op-surface scenes whose means, depths and areas are chosen"""
    rng = np.random.default_rng(seed)
    return (np.tile(np.float32([0.05, 0.01, 0.05]), (C, N, 1)), rng.uniform(0.05, 0.6, (C, N)).astype(np.float32),
            rng.uniform(0, 1, (C, N, 3)).astype(np.float32))


def run_batch(H, W, us, ci, al, depths, col, areas, capacity=False, rgbd=False):
    """ops.splat_batch on device copies -> (outputs, depths and areas after the in-place culls)"""
    d, a = t(depths), t(areas, torch.int32)
    out = ops.splat_batch(H, W, t(us), t(ci), t(al), d, t(col), a, capacity=capacity, rgbd=rgbd)
    return out, d, a


def check_cameras(out, d, a, bins, N, T):
    """camera c's P, tile ranges [c T, (c+1) T), patch list (ids c N + n -> n) and in-place culls against
    its own oracle binning (P, ranges, gsid, keys, depths, areas), bit for bit"""
    ranges, gsid = n(out[3]), n(out[4])
    assert gsid.size == sum(b[0] for b in bins)
    off = 0
    for c, (P, r, g, _, d_or, a_or) in enumerate(bins):
        assert np.array_equal(n(d[c]).view(np.int32), d_or.view(np.int32)), "camera %d: depth cull differs" % c
        assert np.array_equal(n(a[c]), a_or), "camera %d: areas cull differs" % c
        want = np.where((r[:, 1] > r[:, 0])[:, None], r + off, 0)
        assert np.array_equal(ranges[c * T:(c + 1) * T], want), "camera %d: tile ranges differ" % c
        assert np.array_equal(gsid[off:off + P] - c * N, g), "camera %d: patch list differs" % c
        off += P


# ---------------------------------------------------------------- (a) every tall-frame key plan
PLANS_REACHED = {}


@pytest.mark.parametrize("name", list(BATCH_PLANS))
def test_tall_frame_key_plans(name):
    H, W, C, T, us, depths, areas, far = batch_plan_scene(name)
    N = us.shape[1]
    bins = camera_bins(H, W, us, depths, areas)
    keys = tall_keys(bins, T)
    dk = int((keys & np.uint64(0xFFFFFFFF)).max())
    p = key_plan(tall_height(C, H), W, dk)
    PLANS_REACHED[name] = (widths(keys, C * T), plan_shape(p))
    assert (p["tbits"],) + plan_shape(p) == (BATCH_PLANS[name][3][0],) + BATCH_PLANS[name][3][2:]
    ci, al, col = fillers(C, N, seed=len(name))
    exact, d, a = run_batch(H, W, us, ci, al, depths, col, areas)
    check_cameras(exact, d, a, bins, N, T)
    run_batch(H, W, us, ci, al, depths, col, areas, capacity=True)  # learns the bounds (exact path)
    before = dict(ops.CAPACITY_STATS)
    cap, d2, a2 = run_batch(H, W, us, ci, al, depths, col, areas, capacity=True)
    assert ops.CAPACITY_STATS["capacity_frames"] == before["capacity_frames"] + 1, "frame was redone"
    for what, x, y in zip(("image", "contrib", "final_tau", "ranges", "gsid"), exact, cap):
        assert same(x, y), "capacity path differs from the exact path: " + what
    assert same(d, d2) and same(a, a2)
    print("tall plan %-15s (tbits, dbits) %s  %s" % (name, PLANS_REACHED[name][0], PLANS_REACHED[name][1]))


# ---------------------------------------------------------------- (b) the tall frame's row limit
def check_frame_planes(out, c, ref):
    """camera c's planes against the oracle's, at test_gpu_parity's bounds"""
    amb = ref["ambiguous"]
    assert amb.mean() < 5e-3
    err = np.abs(n(out[0][c]).astype(np.float64) - ref["image"]).max(axis=0)
    assert err[~amb].max(initial=0) <= 5e-5 and err.max(initial=0) <= 1e-2, c
    assert np.array_equal(n(out[1][c])[~amb], ref["contrib"][~amb]), c
    assert np.abs(n(out[2][c]).astype(np.float64) - ref["final_tau"])[~amb].max(initial=0) <= 1e-5, c


@pytest.mark.parametrize("C,H,W", ROW_LIMIT)
def test_tall_frame_row_limit(C, H, W):
    need_free_memory(2 << 30)
    s = row_limit_scene(C, H, W, seed=C)
    N = s["us"].shape[1]
    T = ((W + 15) // 16) * ((H + 15) // 16)
    assert tall_height(C, H) // 16 in (65535, 65472)
    out, d, a = run_batch(H, W, s["us"], s["cinv2ds"], s["alphas"], s["depths"], s["colors"], s["areas"])
    refs, bins = [], []
    for c in range(C):
        dc, ac = s["depths"][c].copy(), s["areas"][c].copy()
        ref = orc.splat(H, W, s["us"][c], s["cinv2ds"][c], s["alphas"][c], dc, s["colors"][c], ac)
        bins.append((ref["P"], ref["ranges"], ref["gsid"], ref["keys"], dc, ac))
        refs.append(ref)
    check_cameras(out, d, a, bins, N, T)
    for c in range(C):
        check_frame_planes(out, c, refs[c])
    for c in (0, C - 1):  # the single-camera call's bits
        one = ops.splat(H, W, *(t(s[k][c]) for k in ("us", "cinv2ds", "alphas", "depths", "colors")),
                        t(s["areas"][c], torch.int32))
        for i in range(3):
            assert same(out[i][c], one[i]), (c, i)
        assert np.array_equal(n(one[4]), bins[c][2])
    del out
    torch.cuda.empty_cache()


# ---------------------------------------------------------------- (c) the batch capacity path
@pytest.mark.parametrize("rgbd", [False, True], ids=["colour", "rgbd"])
@pytest.mark.parametrize("layout", ["narrow", "64bit"])
def test_batch_capacity_bounds_and_outgrown_plan(layout, rgbd):
    """P_cap == P: served without a redo; P_cap == P - 1: redone the exact way; then a batch whose depth
    keys need more bits than the plan learnt from the previous one: redone.  Every frame is the exact one."""
    H, W, us, dA, dB, areas = capacity_scene(layout)
    C, N = us.shape[:2]
    T = ((W + 15) // 16) * ((H + 15) // 16)
    key = ("batch", torch.device(DEV).index, C, H, W, N)
    ci, al, col = fillers(C, N, seed=5)

    def frame(dep, capacity):
        return run_batch(H, W, us, ci, al, dep, col, areas, capacity=capacity, rgbd=rgbd)

    def identical(x, y, what):
        assert len(x[0]) == len(y[0]) == (7 if rgbd else 5)
        for i, (p, q) in enumerate(zip(x[0], y[0])):
            assert same(p, q), (what, i)
        assert same(x[1], y[1]) and same(x[2], y[2]), what

    bA = camera_bins(H, W, us, dA, areas)
    exactA = frame(dA, False)
    check_cameras(*exactA, bA, N, T)
    P = sum(b[0] for b in bA)
    dk_cap = ops._next_capacity(P, int((tall_keys(bA, T) & np.uint64(0xFFFFFFFF)).max()))[1]
    for P_cap, redo in ((P, False), (P - 1, True)):
        ops._CAPACITY[key] = (P_cap, dk_cap)
        before = dict(ops.CAPACITY_STATS)
        out = frame(dA, True)
        assert ops.CAPACITY_STATS["outgrown"] == before["outgrown"] + int(redo), P_cap
        assert ops.CAPACITY_STATS["capacity_frames"] == before["capacity_frames"] + int(not redo), P_cap
        identical(exactA, out, "P_cap = %d" % P_cap)
    exactB = frame(dB, False)
    check_cameras(*exactB, camera_bins(H, W, us, dB, areas), N, T)
    ops._CAPACITY.pop(key, None)
    frame(dA, True)  # learns from batch A
    assert ops._CAPACITY[key][1] == dk_cap
    before = dict(ops.CAPACITY_STATS)
    outB = frame(dB, True)
    assert ops.CAPACITY_STATS["outgrown"] == before["outgrown"] + 1
    identical(exactB, outB, "outgrown plan")
    torch.cuda.synchronize()


# ---------------------------------------------------------------- (d) the batch backward rasterizers per entry
def stack_scenes(names):
    """test_gpu_raster_rows scenes, one per camera, padded to one N with rows culled by depth
    -> (the per-camera host arrays (us, ci, alphas, depths, colors, areas), seeds)"""
    cams, seeds = [], []
    for name in names:
        (_, _, *x), seed = scene_inputs(name)
        cams.append([n(v) for v in x])
        seeds.append(seed)
    N = max(len(c[0]) for c in cams)
    pad = (np.float32(0), np.float32([1, 0, 1]), np.float32(0.5), np.float32(-1), np.float32(0), np.int32(0))
    out = []
    for k in range(6):
        rows = []
        for c in cams:
            v = c[k].reshape(len(c[0]), -1) if k != 2 and k != 3 else c[k].reshape(-1)
            fill = np.broadcast_to(pad[k], (N - len(v),) + v.shape[1:])
            rows.append(np.concatenate([v, fill]).astype(v.dtype))
        out.append(np.stack(rows))
    return out, seeds


def rows_per_camera(H, W, cams, seeds, labels, rgbd, records=None):
    """splat_batch, splatB_batch (records given or re-packed) and each camera's slice of the moment rows
    (and dL/dz) against the oracle's rows on that camera's own fp32 inputs"""
    us, ci, al, d, col, ar = cams
    C, N = us.shape[:2]
    T = ((W + 15) // 16) * ((H + 15) // 16)
    out, dd, ad = run_batch(H, W, us, ci, al, d, col, ar, rgbd=rgbd)
    ups = []
    for c in range(C):
        rng = np.random.default_rng(seeds[c] + 101)
        ups.append((upstream_gradient(W, H, seeds[c] + c) * np.float32(3.0 * W * H),
                    (rng.normal(size=(H, W)) / max(float(np.abs(d[c][d[c] > 0]).max(initial=1.0)), 1.0)).astype(
                        np.float32), rng.normal(size=(H, W)).astype(np.float32)))
    dl = t(np.stack([u[0] for u in ups]))
    kw = dict(dloss_ddepth=t(np.stack([u[1] for u in ups])), dloss_dalpha=t(np.stack([u[2] for u in ups]))) \
        if rgbd else {}
    res = ops.splatB_batch(H, W, t(us), t(ci), t(al), dd, t(col), out[1], out[2], out[3], out[4], dl, records=records,
                           **kw)
    mom, dz = (res[0], res[1]) if rgbd else (res, None)
    kernel = "k_draw_bwd_rgbd_batch" if rgbd else "k_draw_bwd_batch"
    bins = []
    for c in range(C):
        dc, ac = d[c].copy(), ar[c].copy()
        if rgbd:
            fwd = orgbd.splat_rgbd(H, W, us[c], ci[c], al[c], dc, col[c], ac)
            ref = orgbd.splat_backward_rgbd_rows(H, W, us[c], ci[c], al[c], col[c], fwd["z"], fwd, *ups[c])
        else:
            fwd = orc.splat(H, W, us[c], ci[c], al[c], dc, col[c], ac)
            ref = oabs.splat_backward_abs_rows(H, W, us[c], ci[c], al[c], col[c], fwd, ups[c][0])
        bins.append((fwd["P"], fwd["ranges"], fwd["gsid"], fwd["keys"], dc, ac))
        check_flagged(ref, fwd["gsid"])
        scene = "cam %d/%d %s" % (c, C, labels[c])
        check_moments(mom[c * N:(c + 1) * N], ref, kernel, scene)
        if rgbd:
            check(dz[c * N:(c + 1) * N], ref["ddepths"], ref["ddepths_abs"], ref["ddepths_maha"], ref["ddepths_amb"],
                  kernel, scene, "ddepths")
    check_cameras(out, dd, ad, bins, N, T)


# (frame W, H: not multiples of 16, so every frame has pad rows), one scene per camera
BWD_BATCHES = {
    2: (401, 307, ["huge_needle", "boundary"]),
    5: (255, 131, ["frame_2000_255_131", "boundary", "clamp", "huge_needle", "frame_40_17_9"]),
}


@pytest.mark.parametrize("rgbd", [False, True], ids=["colour", "rgbd"])
@pytest.mark.parametrize("C", list(BWD_BATCHES))
def test_batch_backward_rows_per_entry(C, rgbd):
    W, H, names = BWD_BATCHES[C]
    cams, seeds = stack_scenes(names)
    rows_per_camera(H, W, cams, seeds, names, rgbd)


def posed_batch(W, H, N, C, seed):
    """a synthetic scene at W x H and C pinhole cameras with their own poses and intrinsics"""
    from easygaussiansplatting_b200.scene import ring_camera, synthetic_scene
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=seed)
    cams = []
    for c in range(C):
        R, tc, tw = ring_camera(c, C, radius=0.3)
        cams.append(Camera(W, H, sc["fx"] * (1.0 + 0.04 * c), sc["fy"] * (1.0 + 0.03 * c), sc["cx"] + 0.7 * c,
                           sc["cy"] - 0.4 * c, t(R), t(tc), t(tw)))
    return {k: t(sc[k]) for k in ("pws", "shs", "scales", "rots", "alphas")}, cams


@pytest.mark.parametrize("rgbd", [False, True], ids=["colour", "rgbd"])
def test_batch_backward_rows_records_given_and_repacked(rgbd):
    """three posed cameras through preprocess_batch at 255x131: splatB_batch on the forward's records and
    on records it packs again, per entry against the oracle"""
    p, cams = posed_batch(255, 131, 2000, 3, seed=3)
    pre = ops.preprocess_batch(p["pws"], p["rots"], p["scales"], p["shs"], cams, p["alphas"])
    C, N = pre[0].shape[:2]
    host = [n(pre[0]), n(pre[1]), np.tile(n(p["alphas"]), (C, 1)), n(pre[3]), n(pre[2]), n(pre[4])]
    for records in (pre[5], None):
        label = "posed, records given" if records is not None else "posed, re-packed"
        rows_per_camera(131, 255, host, [3, 4, 5], [label] * C, rgbd, records=records)


# ---------------------------------------------------------------- (e) every camera model against fp64
MODELS = [("ortho", None), ("fisheye", COLMAP_LIKE_FISHEYE_K), ("opencv", COLMAP_LIKE_OPENCV[0] + COLMAP_LIKE_OPENCV[1])]


def model_scene(model, k, N, W, H, seed):
    """camera_model_scene (opencv: with its tangential coefficients) seen from a general pose"""
    if model == "opencv":
        sc = camera_model_scene(N, W, H, "opencv", k[:2], sh_dim=12, seed=seed, tangential_coeffs=k[2:])
    else:
        sc = camera_model_scene(N, W, H, model, k, sh_dim=12, seed=seed)
    a, b = 0.1, -0.05
    Ry = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    Rx = np.array([[1, 0, 0], [0, np.cos(b), -np.sin(b)], [0, np.sin(b), np.cos(b)]])
    R, tr = Ry @ Rx, np.array([0.1, -0.05, 0.2])
    sc["pws"] = np.ascontiguousarray((sc["pws"].astype(np.float64) - tr) @ R, np.float32)
    sc["Rcw"], sc["tcw"] = R, tr
    return sc


def model_cameras(sc, model, k, C, W, H, aa):
    """C cameras a few degrees and centimetres apart, with their own intrinsics and lens coefficients
    -> (Camera list, the oracle's camera dicts, the oracle's lens k per camera)"""
    cams, camd, ks = [], [], []
    for c in range(C):
        a, b = 0.02 * c, -0.015 * c
        D = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]) @ \
            np.array([[np.cos(b), -np.sin(b), 0], [np.sin(b), np.cos(b), 0], [0, 0, 1]])
        R = (D @ sc["Rcw"]).astype(np.float32)
        tc = (D @ sc["tcw"] + np.array([0.01 * c, -0.005 * c, 0.02 * c])).astype(np.float32)
        tw = (-(R.astype(np.float64).T @ tc.astype(np.float64))).astype(np.float32)
        fx, fy = sc["fx"] * (1.0 + 0.03 * c), sc["fy"] * (1.0 + 0.02 * c)
        cx, cy = sc["cx"] + 1.5 * c, sc["cy"] - 1.0 * c
        kw, kc = {}, None
        if model == "fisheye":
            kc = tuple(x * (1.0 + 0.1 * c) for x in k)
            kw["radial_coeffs"] = kc
        elif model == "opencv":
            kc = tuple(x * (1.0 + 0.1 * c) for x in k[:2]) + tuple(x * (1.0 - 0.2 * c) for x in k[2:])
            kw.update(radial_coeffs=kc[:2], tangential_coeffs=kc[2:])
        cams.append(Camera(W, H, fx, fy, cx, cy, t(R), t(tc), t(tw), antialiased=aa, camera_model=model, **kw))
        camd.append(dict(Rcw=R, tcw=tc, twc=tw, fx=fx, fy=fy, cx=cx, cy=cy, width=W, height=H))
        ks.append(kc)
    return cams, camd, ks


@pytest.mark.parametrize("rgbd", [False, True], ids=["colour", "rgbd"])
@pytest.mark.parametrize("aa", [False, True], ids=["plain", "aa"])
@pytest.mark.parametrize("model,k", MODELS, ids=[m for m, _ in MODELS])
def test_camera_models_through_the_batch_against_oracle(model, k, aa, rgbd):
    """planes 1e-4 (image) and 2e-4 (depth, alpha) off the oracle's ambiguous pixels; summed map gradients
    and dL/du per camera 2e-4 of max |ref| on the rows the oracle does not flag.  The oracle renders on the
    batch's own fp32 per-Gaussian rows, which under fisheye are not the single call's bits (DESIGN 3.21)."""
    W, H, N, C = 93, 61, 600, 3 if model != "opencv" else 4
    sc = model_scene(model, k, N, W, H, seed=5)
    cams, camd, ks = model_cameras(sc, model, k, C, W, H, aa)
    P = {q: t(sc[q]).requires_grad_() for q in ("pws", "shs", "scales", "rots")}
    al = t(sc["alphas"][:, None]).requires_grad_()
    us = torch.zeros((C, N, 2), device=DEV, requires_grad=True)
    rng = np.random.default_rng(9)
    ups = [(upstream_gradient(W, H, 3 + c) * np.float32(3.0 * W * H), rng.normal(size=(H, W)).astype(np.float32) * 0.1,
            rng.normal(size=(H, W)).astype(np.float32)) for c in range(C)]
    F = GSFunctionFusedBatchRGBD if rgbd else GSFunctionFusedBatch
    outs = F.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us, cams)
    loss = sum((outs[0][c] * t(dl)).sum() + ((outs[1][c] * t(dld)).sum() + (outs[2][c] * t(dla)).sum() if rgbd else 0)
               for c, (dl, dld, dla) in enumerate(ups))
    loss.backward()
    pre = ops.preprocess_batch(t(sc["pws"]), t(sc["rots"]), t(sc["scales"]), t(sc["shs"]), cams, t(sc["alphas"]))
    scene = {q: sc[q] for q in ("pws", "rots", "scales", "shs", "alphas")}
    step = ocv.step if model == "opencv" else ocm.step
    refs = []
    for c in range(C):
        drawn = dict(us=n(pre[0][c]), ci=n(pre[1][c]), col=n(pre[2][c]), depths=n(pre[3][c]), areas=n(pre[4][c]),
                     alphas=n(pre[6][c]) if aa else sc["alphas"])
        dl, dld, dla = ups[c]
        o = step(scene, camd[c], rgbd=rgbd, pose=False, aa=aa, filt=None, dl=dl, dld=dld if rgbd else None,
                 dla=dla if rgbd else None, drawn_inputs=drawn, model=model, k=ks[c])
        amb = o["ambiguous"]
        assert amb.mean() < 0.01, (c, amb.mean())
        assert np.abs(n(outs[0][c]) - o["image"]).max(0)[~amb].max() < 1e-4, c
        if rgbd:
            for i, name in ((1, "depth"), (2, "alpha")):
                assert np.abs(n(outs[i][c]) - o[name])[~amb].max() <= 2e-4, (c, name)
        close_rows(n(us.grad[c]), o["grads"]["us"], ~o["flagged"], tol=2e-4, what="dus[%d]" % c)
        refs.append(o)
    rows = ~np.any([o["flagged"] for o in refs], axis=0)
    assert rows.mean() > 0.9
    got = dict(pws=P["pws"].grad, shs=P["shs"].grad, scales=P["scales"].grad, rots=P["rots"].grad, alphas=al.grad)
    for q, g in got.items():
        close_rows(n(g), sum(o["grads"][q].reshape(N, -1) for o in refs), rows, tol=2e-4, what="d" + q)


# ---------------------------------------------------------------- (f) C = 64
@pytest.mark.parametrize("k3,model", [(16, "pinhole"), (4, "opencv")])
def test_64_cameras_against_the_single_camera_loop(k3, model):
    """the GSB_BATCH_MAX_CAMERAS cap at 83x61 (partial tiles): planes bit for bit and gradients to 1e-5 of
    max |g| against 64 single-camera calls; the moment rows of cameras 0 and 63 per entry"""
    C = ops.BATCH_MAX_CAMERAS
    sc, p = batch_params(400, k3, seed=64 + k3)
    cams = batch_cams(sc, C, model)
    from test_gpu_batch import H as BH, W as BW
    N = p["pws"].shape[0]
    g = torch.Generator(device=DEV).manual_seed(k3)
    Gi = torch.randn((C, 3, BH, BW), generator=g, device=DEV)
    leaves = lambda: ({q: p[q].clone().requires_grad_() for q in ("pws", "shs", "scales", "rots")} |
                      {"alphas": p["alphas"][:, None].clone().requires_grad_()})
    L = leaves()
    us = torch.zeros((C, N, 2), device=DEV, requires_grad=True)
    img, mask = GSFunctionFusedBatch.apply(L["pws"], L["shs"], L["alphas"], L["scales"], L["rots"], us, cams)
    (img * Gi).sum().backward()
    S = leaves()
    for c, cam in enumerate(cams):
        u = torch.zeros((N, 2), device=DEV, requires_grad=True)
        i1, m1 = GSFunctionFused.apply(S["pws"], S["shs"], S["alphas"], S["scales"], S["rots"], u, cam)
        (i1 * Gi[c]).sum().backward()
        assert torch.equal(img[c].detach(), i1.detach()) and torch.equal(mask[c], m1), c
        close_max(us.grad[c], u.grad, "dus[%d]" % c)
    for q in ("pws", "shs", "alphas", "scales", "rots"):
        close_max(L[q].grad, S[q].grad, q)
    # per entry: the batch's moment rows of the first and the last camera on the forward's records
    pre = ops.preprocess_batch(p["pws"], p["rots"], p["scales"], p["shs"], cams, p["alphas"])
    out = ops.splat_batch(BH, BW, pre[0], pre[1], p["alphas"], pre[3].clone(), pre[2], pre[4].clone(), records=pre[5])
    mom = ops.splatB_batch(BH, BW, pre[0], pre[1], p["alphas"], pre[3], pre[2], out[1], out[2], out[3], out[4],
                           Gi.contiguous(), records=pre[5])
    for c in (0, C - 1):
        h = [n(pre[0][c]), n(pre[1][c]), n(p["alphas"]), n(pre[3][c]).copy(), n(pre[2][c]), n(pre[4][c]).copy()]
        fwd = orc.splat(BH, BW, h[0], h[1], h[2], h[3], h[4], h[5])
        ref = oabs.splat_backward_abs_rows(BH, BW, h[0], h[1], h[2], h[4], fwd, n(Gi[c]))
        check_flagged(ref, fwd["gsid"])
        check_moments(mom[c * N:(c + 1) * N], ref, "k_draw_bwd_batch", "C64 %s k3=%d cam %d" % (model, k3, c))
