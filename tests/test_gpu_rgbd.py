"""RGB-D rendering on the GPU: `splat_rgbd` / `splatB_rgbd` / `preprocessB(dloss_ddepths=...)` /
GSFunctionFusedRGBD against the fp64 oracle (oracle/rgbd_oracle.c's orc_draw_rgbd and
orc_drawB_rgbd, and the chain with its depth term), and against the colour path they extend.

Tolerances: the colour outputs are bit-identical to `splat`'s; A <= 5e-5 abs and D <= 5e-5 max z
on pixels without a threshold-ambiguous decision (1e-2 / 1e-2 max z on the flagged ones, as for
the image); per-Gaussian gradients <= 1e-4 max|ref| per tensor (5e-3 on threshold-ambiguous
Gaussians)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from oracle import rgbd_oracle as orgbd
from easygaussiansplatting_b200.scene import synthetic_scene, upstream_gradient

from test_gpu_parity import DEV, gaussians_in_tile, n, op_inputs, scene_with_culls, t

pytestmark = pytest.mark.gpu


def ops():
    from easygaussiansplatting_b200 import ops as o
    return o


def preprocess(sc):
    return ops().preprocess(*[t(sc[k]) for k in ("pws", "rots", "scales", "shs", "Rcw", "tcw", "twc")],
                            sc["fx"], sc["fy"], sc["cx"], sc["cy"], sc["width"], sc["height"])


def bound(got, want, amb, name, tol=1e-4, tol_amb=5e-3):
    """per-Gaussian rows: max err / max|ref| <= tol off the ambiguous rows, tol_amb on them"""
    want = np.asarray(want, np.float64).reshape(len(amb), -1)
    err = np.abs(n(got).astype(np.float64).reshape(want.shape) - want).max(axis=1)
    s = np.abs(want).max(initial=1e-30)
    assert err[~amb].max(initial=0) / s <= tol, "%s: normalised max err %.3e" % (name, err[~amb].max() / s)
    assert err.max(initial=0) / s <= tol_amb, "%s: ambiguous-Gaussian err %.3e" % (name, err.max() / s)


def upstream(W, H, seed, zmax):
    rng = np.random.default_rng(seed + 77)
    dl = upstream_gradient(W, H, seed) * (3.0 * W * H)
    dld = (rng.normal(size=(H, W)) / zmax).astype(np.float32)
    dla = rng.normal(size=(H, W)).astype(np.float32)
    return dl, dld, dla


def tile_zmax(H, W, ref):
    """[H,W]: the largest |z| in the patch list of each pixel's tile (0 on empty tiles), from the
    oracle forward's ranges / gsid / z"""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    lens = ref["ranges"][:, 1] - ref["ranges"][:, 0]
    zt = np.zeros(gx * gy)
    np.maximum.at(zt, np.repeat(np.arange(gx * gy), lens), np.abs(ref["z"][ref["gsid"]]))
    return np.repeat(np.repeat(zt.reshape(gy, gx), 16, axis=0), 16, axis=1)[:H, :W]


def check_rgbd(H, W, us_d, ci_d, al_d, d_d, col_d, ar_d, seed=0, records=None, capacity=False, tol_scale=1.0,
               tile_z=False):
    """splat_rgbd (+ splatB_rgbd) against splat / splatB and the oracle.  d_d / ar_d are culled
    in place.  tile_z: D is bounded per pixel by the largest z of its own tile's list instead of
    the frame's (for scenes whose depths span orders of magnitude).
    -> (the seven outputs, the oracle forward, the five gradients)"""
    o = ops()
    us, ci, col, al = n(us_d), n(ci_d), n(col_d), n(al_d)
    d_in, a_in = n(d_d).copy(), n(ar_d).copy()
    d_rgb, a_rgb = d_d.clone(), ar_d.clone()
    rgb = o.splat(H, W, us_d, ci_d, al_d, d_rgb, col_d, a_rgb, records=records)
    out = o.splat_rgbd(H, W, us_d, ci_d, al_d, d_d, col_d, ar_d, records=records, capacity=capacity)
    assert len(out) == 7
    for name, x, y in zip(("image", "contrib", "final_tau", "ranges", "gsid"), rgb, out[:5]):
        assert torch.equal(x, y), name
    assert torch.equal(d_rgb, d_d) and torch.equal(a_rgb, ar_d)
    ref = orgbd.splat_rgbd(H, W, us, ci, al, d_in.copy(), col, a_in.copy(), margin=2e-5 * tol_scale)
    assert np.array_equal(n(out[4]), ref["gsid"])
    amb = ref["ambiguous"]
    zmax = max(float(np.abs(ref["z"][ref["gsid"]]).max(initial=0.0)), 1.0)
    eA = np.abs(n(out[6]).astype(np.float64) - ref["alpha"])
    eD = np.abs(n(out[5]).astype(np.float64) - ref["depth"])
    assert eA[~amb].max(initial=0) <= 5e-5 * tol_scale, "alpha err %.3e" % eA[~amb].max()
    if tile_z:
        eD = eD / np.maximum(tile_zmax(H, W, ref), 1.0)
        assert eD[~amb].max(initial=0) <= 5e-5 * tol_scale, "depth err %.3e of the tile's max z" % eD[~amb].max()
        assert eA.max(initial=0) <= 1e-2 and eD.max(initial=0) <= 1e-2
    else:
        assert eD[~amb].max(initial=0) <= 5e-5 * tol_scale * zmax, "depth err %.3e of %g" % (eD[~amb].max(), zmax)
        assert eA.max(initial=0) <= 1e-2 and eD.max(initial=0) <= 1e-2 * zmax
    # backward: all five per-Gaussian gradients against the oracle
    dl, dld, dla = upstream(W, H, seed, zmax)
    g5 = o.splatB_rgbd(H, W, us_d, ci_d, al_d, d_d, col_d, out[1], out[2], out[3], out[4], t(dl), t(dld), t(dla),
                       records=records)
    *ref5, amb_gs = orgbd.splat_backward_rgbd(H, W, us, ci, al, col, ref["z"], ref, dl, dld, dla, return_ambiguous=True,
                                            margin=2e-5 * tol_scale)
    assert amb_gs.mean() <= 0.01 * tol_scale
    for got, want, name in zip(g5, ref5, ("dus", "dcinv2ds", "dalphas", "dcolors", "ddepths")):
        bound(got, want, amb_gs, name, 1e-4 * tol_scale, 5e-3 * tol_scale)
    return out, ref, g5


@pytest.mark.parametrize("N,W,H", [(3000, 979, 546), (2000, 255, 131), (40, 17, 9), (8, 7, 5), (4001, 320, 200)])
def test_splat_rgbd_and_backward_vs_oracle(N, W, H):
    sc = scene_with_culls(N, W, H, 3, N)
    us, ci, col, d, ar = preprocess(sc)
    check_rgbd(H, W, us, ci, t(sc["alphas"]), d, col, ar, seed=N)


def test_config2_rgbd_vs_oracle():
    """1M Gaussians at 1920x1080 (BASELINE config 2), forward and backward"""
    N, W, H = 1_000_000, 1920, 1080
    sc = synthetic_scene(N, W, H, sh_dim=48, seed=0)
    us, ci, col, d, ar = preprocess(sc)
    check_rgbd(H, W, us, ci, t(sc["alphas"]), d, col, ar, seed=2)


def test_zero_depth_and_alpha_gradients_are_the_colour_backward():
    o = ops()
    N, W, H = 20000, 640, 480
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=5)
    us, ci, col, d, ar = preprocess(sc)
    al = t(sc["alphas"])
    out = o.splat_rgbd(H, W, us, ci, al, d, col, ar)
    dl = t(upstream_gradient(W, H, 5) * (3.0 * W * H))
    z = torch.zeros((H, W), device=DEV)
    g4 = o.splatB(H, W, us, ci, al, d, col, *out[1:5], dl)
    g5 = o.splatB_rgbd(H, W, us, ci, al, d, col, *out[1:5], dl, z, z)
    for a, b in zip(g4, g5[:4]):  # (sums of float atomics: equal to their ordering)
        assert float((a - b).abs().max()) <= 1e-5 * float(a.abs().max())
    assert not bool(g5[4].any())
    m4 = o.splatB(H, W, us, ci, al, d, col, *out[1:5], dl, moments_only=True)
    m5, dz = o.splatB_rgbd(H, W, us, ci, al, d, col, *out[1:5], dl, z, z, moments_only=True)
    assert float((m4 - m5).abs().max()) <= 1e-5 * float(m4.abs().max()) and not bool(dz.any())


def test_tile_entries_clamped_opacity_and_far_depths():
    """whole-tile (<= 32 patches) and four-entry (>= 33) work items with the 32-record chunk edges,
    opacities at and above the 0.99 clamp (the backward's shuffle path), and a third of the tiles
    near 1 km (64-bit sort keys; depth magnitudes ~1e3)"""
    rng = np.random.default_rng(9)
    gx, parts = 8, []
    tiles = [1, 2, 31, 32, 33, 63, 64, 65, 97, 34, 32, 40, 40]
    for i, k in enumerate(tiles):
        p = gaussians_in_tile(i % gx, i // gx, k, rng, alpha=(0.02, 0.3) if k > 32 else (0.05, 0.9),
                              z0=rng.uniform(950.0, 1050.0) if i % 3 == 0 else rng.uniform(1.0, 20.0))
        if i in (9, 10):
            p[2][28:32] = (0.99, np.nextafter(np.float32(0.99), np.float32(1)), 1.0, 1.0)
        parts.append(p)
    # a wide frame pushes the tile index bits so that depth bits + tile bits > 32
    W, H = 16 * 1024, 16 * 8
    out, ref, _ = check_rgbd(H, W, *op_inputs(parts), seed=9)
    lens = ref["ranges"][:, 1] - ref["ranges"][:, 0]
    assert sorted(lens[lens > 0].tolist()) == sorted(tiles)
    depth_bits = int((ref["keys"] & 0xFFFFFFFF).max()).bit_length()
    assert depth_bits >= 20 and depth_bits + (1024 * 8 - 1).bit_length() > 32
    assert float(out[5].max()) > 500.0


def test_capacity_path_and_overflow_fallback():
    o = ops()
    N, W, H = 30000, 800, 600
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=8)
    us, ci, col, d, ar = preprocess(sc)
    al = t(sc["alphas"])
    key = (torch.device(DEV).index or 0, H, W, N)
    o._CAPACITY.pop(key, None)
    exact = check_rgbd(H, W, us, ci, al, d.clone(), col, ar.clone(), seed=8, capacity=True)[0]
    assert key in o._CAPACITY
    before = dict(o.CAPACITY_STATS)
    cap = o.splat_rgbd(H, W, us, ci, al, d.clone(), col, ar.clone(), capacity=True)
    assert o.CAPACITY_STATS["capacity_frames"] == before["capacity_frames"] + 1
    for x, y in zip(exact, cap):
        assert torch.equal(x, y)
    o._CAPACITY[key] = (64, o._CAPACITY[key][1])  # far too few patch slots: redone the exact way
    over = o.splat_rgbd(H, W, us, ci, al, d.clone(), col, ar.clone(), capacity=True)
    assert o.CAPACITY_STATS["outgrown"] == before["outgrown"] + 1
    for x, y in zip(exact, over):
        assert torch.equal(x, y)


def test_empty_scene_and_no_patches():
    o = ops()
    W, H = 100, 70
    e = torch.empty((0, 2), device=DEV)
    out = o.splat_rgbd(H, W, e, torch.empty((0, 3), device=DEV), torch.empty(0, device=DEV),
                       torch.empty(0, device=DEV), torch.empty((0, 3), device=DEV),
                       torch.empty((0, 2), dtype=torch.int32, device=DEV))
    assert out[4].numel() == 0 and not bool(out[5].any()) and not bool(out[6].any())
    g = o.splatB_rgbd(H, W, e, torch.empty((0, 3), device=DEV), torch.empty(0, device=DEV), torch.empty(0, device=DEV),
                      torch.empty((0, 3), device=DEV), *out[1:5], torch.zeros((3, H, W), device=DEV),
                      torch.ones((H, W), device=DEV), torch.ones((H, W), device=DEV))
    assert g[4].shape == (0,)
    # every Gaussian behind the camera: P = 0, D = A = 0, all gradients 0
    sc = synthetic_scene(500, W, H, sh_dim=3, seed=1)
    sc["pws"][:, 2] = -1.0
    us, ci, col, d, ar = preprocess(sc)
    al = t(sc["alphas"])
    out = o.splat_rgbd(H, W, us, ci, al, d, col, ar)
    assert out[4].numel() == 0 and not bool(out[5].any()) and not bool(out[6].any())
    g = o.splatB_rgbd(H, W, us, ci, al, d, col, *out[1:5], torch.ones((3, H, W), device=DEV),
                      torch.ones((H, W), device=DEV), torch.ones((H, W), device=DEV))
    assert all(not bool(x.any()) for x in g)


def test_offset_upstream_views():
    """dL/dD and dL/dA as contiguous views one float into their storage (scalar loads): the same
    gradients (the moment rows and dL/dz are sums of float atomics, so equal to their ordering)"""
    o = ops()
    N, W, H = 20001, 979, 546
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=3)
    us, ci, col, d, ar = preprocess(sc)
    al = t(sc["alphas"])
    out = o.splat_rgbd(H, W, us, ci, al, d, col, ar)
    dl, dld, dla = upstream(W, H, 3, 12.0)

    def shifted(x):
        v = torch.empty(x.numel() + 1, device=DEV)[1:].view(x.shape)
        v.copy_(x)
        assert v.data_ptr() % 16 == 4
        return v

    a = o.splatB_rgbd(H, W, us, ci, al, d, col, *out[1:5], t(dl), t(dld), t(dla))
    b = o.splatB_rgbd(H, W, us, ci, al, d, col, *out[1:5], shifted(t(dl)), shifted(t(dld)), shifted(t(dla)))
    for x, y in zip(a, b):
        assert torch.equal(x != 0, y != 0)
        assert float((x - y).abs().max()) <= 1e-5 * float(x.abs().max())


def test_misaligned_depth_and_alpha_planes_are_refused():
    from easygaussiansplatting_b200 import _lib
    o = ops()
    N, W, H = 500, 64, 48
    sc = synthetic_scene(N, W, H, sh_dim=3, seed=1)
    us, ci, col, d, ar = preprocess(sc)
    al = t(sc["alphas"])
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    bin_bytes = lib.gsb_splat_bin_workspace_bytes(N)
    bin_ws = torch.empty(bin_bytes, dtype=torch.uint8, device=DEV)
    P, dk = C.c_int64(0), C.c_uint32(0)
    _lib.check(lib.gsb_splat_bin(H, W, N, us.data_ptr(), d.data_ptr(), ar.data_ptr(), bin_ws.data_ptr(), bin_bytes,
                                 C.byref(P), C.byref(dk), st), lib)
    P = int(P.value)
    ws_bytes = lib.gsb_splat_workspace_bytes(N, H, W, P)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
    T = ((W + 15) // 16) * ((H + 15) // 16)
    img, con, ft = torch.empty((3, H, W), device=DEV), torch.empty((H, W), dtype=torch.int32, device=DEV), \
        torch.empty((H, W), device=DEV)
    rg, gsid = torch.empty((T, 2), dtype=torch.int32, device=DEV), torch.empty(max(P, 1), dtype=torch.int32, device=DEV)
    ok = torch.empty((H, W), device=DEV)
    bad = torch.empty(H * W + 1, device=DEV)[1:].view(H, W)

    def render(dimg, aimg):
        return lib.gsb_splat_render_rgbd(H, W, N, P, dk.value, us.data_ptr(), ci.data_ptr(), al.data_ptr(),
                                         d.data_ptr(), col.data_ptr(), None, bin_ws.data_ptr(), ws.data_ptr(), ws_bytes,
                                         img.data_ptr(), con.data_ptr(), ft.data_ptr(), rg.data_ptr(), gsid.data_ptr(),
                                         dimg.data_ptr(), aimg.data_ptr(), st)

    assert render(ok, torch.empty((H, W), device=DEV)) == 0
    torch.cuda.synchronize()
    for args in ((bad, ok), (ok, bad)):
        assert render(*args) != 0 and b"misaligned" in lib.gsb_last_error()
    status = torch.zeros(4, dtype=torch.int32).pin_memory()
    rc = lib.gsb_splat_forward_rgbd(H, W, N, us.data_ptr(), ci.data_ptr(), al.data_ptr(), d.data_ptr(), col.data_ptr(),
                                    ar.data_ptr(), None, P + 16, dk.value, bin_ws.data_ptr(), bin_bytes, ws.data_ptr(),
                                    ws_bytes, img.data_ptr(), con.data_ptr(), ft.data_ptr(), rg.data_ptr(),
                                    gsid.data_ptr(), status.data_ptr(), ok.data_ptr(), bad.data_ptr(), st)
    assert rc != 0 and b"misaligned" in lib.gsb_last_error()
    torch.cuda.synchronize()


def test_backward_never_reads_records_without_depth():
    """the records splatB_rgbd uses carry z: the ones `preprocess(alphas=...)` returns, those
    `splat` packs (looked up only while `depths` is unchanged), or a re-pack from `depths`"""
    o = ops()
    N, W, H = 20000, 640, 480
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=12)
    P7 = [t(sc[k]) for k in ("pws", "rots", "scales", "shs", "Rcw", "tcw", "twc")]
    al = t(sc["alphas"])
    us, ci, col, d, ar, recs = o.preprocess(*P7, sc["fx"], sc["fy"], sc["cx"], sc["cy"], W, H, alphas=al)
    assert torch.equal(recs[:, 11], d)  # the depth word
    d0 = d.clone()
    ref_out, _, ref_g = check_rgbd(H, W, us, ci, al, d, col, ar, seed=12, records=recs)
    dl, dld, dla = upstream(W, H, 12, float(d0.max()))
    # records packed by the colour `splat`, found through gsid_per_patch
    d1, ar1 = d0.clone(), o.preprocess(*P7, sc["fx"], sc["fy"], sc["cx"], sc["cy"], W, H)[4]
    out = o.splat(H, W, us, ci, al, d1, col, ar1)
    assert o._cached_records(out[4], (us, ci, al, col, d1)) is not None
    g_cached = o.splatB_rgbd(H, W, us, ci, al, d1, col, *out[1:5], t(dl), t(dld), t(dla))
    # an in-place edit of depths invalidates them for the RGB-D backward (not for the colour one)
    d1.add_(0.0)
    assert o._cached_records(out[4], (us, ci, al, col, d1)) is None
    assert o._cached_records(out[4], (us, ci, al, col)) is not None
    g_repacked = o.splatB_rgbd(H, W, us, ci, al, d1, col, *out[1:5], t(dl), t(dld), t(dla))
    g_given = o.splatB_rgbd(H, W, us, ci, al, d1, col, *out[1:5], t(dl), t(dld), t(dla), records=recs)
    for a, b, c in zip(g_cached, g_repacked, g_given):
        s = float(a.abs().max())
        assert float((a - b).abs().max()) <= 1e-5 * s and float((a - c).abs().max()) <= 1e-5 * s
    assert float(g_cached[4].abs().max()) > 0


@pytest.mark.parametrize("k3", [1, 4, 9, 16])
def test_gsfunction_fused_rgbd_vs_oracle_chain(k3):
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFusedRGBD
    N, W, H = 4001, 320, 200
    sc = scene_with_culls(N, W, H, 3 * k3, 40 + k3)
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]))
    params = {k: t(sc[k]).requires_grad_(True) for k in ("pws", "shs", "alphas", "scales", "rots")}
    us_slot = torch.zeros((N, 2), device=DEV, requires_grad=True)
    image, depth, alpha, mask = GSFunctionFusedRGBD.apply(params["pws"], params["shs"], params["alphas"],
                                                          params["scales"], params["rots"], us_slot, cam)
    dl, dld, dla = upstream(W, H, k3, 12.0)
    ((image * t(dl)).sum() + (depth * t(dld)).sum() + (alpha * t(dla)).sum()).backward()
    # the oracle: stages with Jacobians, RGB-D compositing, its backward and the chain
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    us, pcs, depths, Ju = orc.project(sc["pws"], sc["Rcw"], sc["tcw"], sc["fx"], sc["fy"], sc["cx"], sc["cy"])
    d32 = f32(depths)
    c3, J3r, J3s = orc.compute_cov3d(sc["rots"], sc["scales"], d32)
    c2, J2c, J2p = orc.compute_cov2d(f32(c3), f32(pcs), sc["Rcw"], d32, sc["fx"], sc["fy"], W, H)
    col, Jcs, Jcp = orc.sh2color(sc["shs"], sc["pws"], sc["twc"])
    ci, areas, Jci = orc.inverse_cov2d(f32(c2), d32)
    # the tile rectangles are integer decisions on the fp32 radius (ceil(3 sqrt(.))): bin the oracle
    # with the fused forward's own radii, so both composite the same patch lists
    areas = np.ascontiguousarray(n(preprocess(sc)[4]))
    # the fused forward's u / conic are its own fp32 values (1e-4-level relative differences to the
    # oracle stages, test_fused_math_cpu.py): threshold decisions that close are flagged ambiguous
    margin = 5e-4
    ref = orgbd.splat_rgbd(H, W, us, ci, sc["alphas"], d32, col, areas, margin=margin)
    assert ref["ambiguous"].mean() < 0.02
    assert np.abs(n(alpha) - ref["alpha"])[~ref["ambiguous"]].max() <= 1e-4
    assert mask.shape == (N,) and mask.dtype == torch.bool
    *g5, amb = orgbd.splat_backward_rgbd(H, W, us, ci, sc["alphas"], col, ref["z"], ref, dl, dld, dla,
                                       return_ambiguous=True, margin=margin)
    assert amb.mean() < 0.05
    chain = orc.chain_backward(sc["Rcw"], *g5[:4], Ju, J3r, J3s, J2c, J2p, Jcs, Jcp, Jci)
    want = {"pws": chain["pws"] + orgbd.chain_depth(sc["Rcw"], g5[4], ref["z"]), "shs": chain["shs"],
            "alphas": np.asarray(g5[2]).reshape(-1), "scales": chain["scales"], "rots": chain["rots"]}
    for k in want:
        # (the fused recomputation in fp32 against the fp64 chain: test_gpu_fused_oracle.py's bound)
        bound(params[k].grad, want[k], amb, k, tol=2e-4, tol_amb=5e-3)
    bound(us_slot.grad, g5[0].reshape(N, 2), amb, "us", tol=2e-4)


def test_depth_only_optimisation_descends():
    """L1 on D against a hidden scene's depth, pws and scales trainable: 100 Adam steps at 320x240"""
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFusedRGBD
    N, W, H = 3000, 320, 240
    sc = synthetic_scene(N, W, H, sh_dim=3, seed=21)
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]))
    fixed = {k: t(sc[k]) for k in ("shs", "alphas", "rots")}
    us_slot = torch.zeros((N, 2), device=DEV, requires_grad=True)
    with torch.no_grad():
        _, target, _, _ = GSFunctionFusedRGBD.apply(t(sc["pws"]), fixed["shs"], fixed["alphas"], t(sc["scales"]),
                                                    fixed["rots"], us_slot, cam)
    rng = np.random.default_rng(3)
    pws = t(sc["pws"] * (1.0 + 0.04 * rng.normal(size=(N, 1)))).requires_grad_(True)  # along the viewing rays
    scales = t(sc["scales"] * np.exp(0.2 * rng.normal(size=(N, 3)))).requires_grad_(True)
    opt = torch.optim.Adam([pws, scales], lr=5e-3)
    losses = []
    for _ in range(100):
        opt.zero_grad()
        _, depth, _, _ = GSFunctionFusedRGBD.apply(pws, fixed["shs"], fixed["alphas"], scales, fixed["rots"],
                                                   us_slot, cam)
        loss = (depth - target).abs().mean()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert all(np.isfinite(losses))
    assert np.mean(losses[-5:]) < 0.6 * losses[0], losses[::10]
