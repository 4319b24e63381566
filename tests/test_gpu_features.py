"""Feature rendering on the GPU: `splat_features` / `splatB_features` / GSFunctionFusedFeatures and the
density rebuild of per-Gaussian features.

1. Identities against outputs already verified elsewhere: colours as features give the image bit for
   bit, z and 1 the RGB-D depth and alpha planes bit for bit; with dL/dF = dL/dgamma the added moment
   rows and dL/dfeatures are splatB's (fp32 atomic-order tolerance).
2. The fp64 feature oracle (oracle/feature_oracle.py): the map to 1e-4 max|f| off threshold-ambiguous
   pixels; the gradients to 1e-4 max|g| per tensor off ambiguous Gaussians (5e-3 on them), as
   test_gpu_rgbd.py -- for D from 1 to 64, odd frame sizes, empty tiles, N = 0, no patches, the
   capacity path and its fallback, features at an odd 4-byte offset.
3. Whole steps through the class against feature_oracle.step_features (plain, AA, filter, both).
4. The skip paths, 5. density with extra=("features",), 6. a short training run."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import feature_oracle as ofe
from oracle import step_oracle as ost
from easygaussiansplatting_b200.scene import synthetic_scene, upstream_gradient

from test_gpu_parity import DEV, gaussians_in_tile, n, op_inputs, scene_with_culls, t
from test_gpu_rgbd import preprocess
from test_gpu_step_matrix import _camera, bits, check_grads, check_planes, drawn_frame, matrix_scene

pytestmark = pytest.mark.gpu


def ops():
    from easygaussiansplatting_b200 import ops as o
    return o


def frame(sc, W, H, capacity=False):
    """preprocess + splat of a scene dict -> ((us, ci, al, col, d, ar, records), splat's five outputs)"""
    o = ops()
    al = t(sc["alphas"])
    pre = o.preprocess(*[t(sc[k]) for k in ("pws", "rots", "scales", "shs", "Rcw", "tcw", "twc")], sc["fx"], sc["fy"],
                       sc["cx"], sc["cy"], W, H, alphas=al)
    us, ci, col, d, ar, recs = pre
    out = o.splat(H, W, us, ci, al, d, col, ar, records=recs, capacity=capacity)
    return (us, ci, al, col, d, ar, recs), out


def feats(N, D, seed):
    return np.random.default_rng(seed).normal(size=(N, D)).astype(np.float32)


def moments_to_grads(mom, ci):
    """the conversion of moment rows 0-5 (k_finalize_grads' formulas) in fp64 -> du[N,2], dconic[N,3], dalpha[N]"""
    m = n(mom).astype(np.float64)
    c = n(ci).astype(np.float64)
    A, B, Cc = c[:, 0], c[:, 1], c[:, 2]
    du = -np.stack([A * m[:, 0] + B * m[:, 1], B * m[:, 0] + Cc * m[:, 1]], 1)
    dc = np.stack([-0.5 * m[:, 2], -m[:, 3], -0.5 * m[:, 4]], 1)
    return du, dc, m[:, 5]


def bound(got, want, amb, name, tol=1e-4, tol_amb=5e-3):
    want = np.asarray(want, np.float64).reshape(len(amb), -1)
    err = np.abs(np.asarray(got, np.float64).reshape(want.shape) - want).max(axis=1)
    s = np.abs(want).max(initial=1e-30)
    assert err[~amb].max(initial=0) / s <= tol, "%s: normalised max err %.3e" % (name, err[~amb].max() / s)
    assert err.max(initial=0) / s <= tol_amb, "%s: ambiguous-Gaussian err %.3e" % (name, err.max() / s)


def check_features(H, W, inp, out, f, seed=0, records=None):
    """splat_features + splatB_features on a drawn frame against the oracle on the same fp32 values"""
    o = ops()
    us, ci, al, col, d, ar, _ = inp
    fd = f if isinstance(f, torch.Tensor) else t(f)
    f64 = n(fd)
    N, D = f64.shape
    fmap = o.splat_features(H, W, fd, out[1], out[3], out[4], records=records, us=us, cinv2ds=ci, alphas=al, colors=col)
    assert tuple(fmap.shape) == (D, H, W)
    ref = ofe.splat_features(H, W, n(us), n(ci), n(al), n(d), n(ar), f64)
    assert np.array_equal(n(out[4]), ref["gsid"])
    amb = ref["ambiguous"]
    assert amb.mean() < 0.01
    fmax = max(float(np.abs(f64).max(initial=0.0)), 1.0)
    e = np.abs(n(fmap).astype(np.float64) - ref["features"])
    e = e.max(0)
    assert e[~amb].max(initial=0) <= 1e-4 * fmax, "feature map err %.3e" % e[~amb].max()
    assert e.max(initial=0) <= 1e-2 * fmax
    dF = np.random.default_rng(seed + 5).normal(size=(D, H, W)).astype(np.float32)
    mom, dfeat = o.splatB_features(H, W, fd, out[1], out[2], out[3], out[4], t(dF), records=records, us=us,
                                   cinv2ds=ci, alphas=al, colors=col)
    assert tuple(dfeat.shape) == (N, D) and not n(mom)[:, 6:].any()
    *refg, amb_gs = ofe.splat_backward_features(H, W, n(us), n(ci), n(al), ref, f64, dF, return_ambiguous=True)
    assert amb_gs.mean() <= 0.01
    du, dc, da = moments_to_grads(mom, ci)
    for got, want, name in zip((du, dc, da, n(dfeat)), refg, ("dus", "dcinv2ds", "dalphas", "dfeatures")):
        bound(got, want, amb_gs, name)
    return fmap, ref, (mom, dfeat)


# ---------------------------------------------------------------- 1. identities
@pytest.mark.parametrize("N,W,H", [(20000, 640, 480), (3000, 979, 546)])
def test_identities_with_the_image_and_the_rgbd_planes(N, W, H):
    o = ops()
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=N)
    inp, out = frame(sc, W, H)
    us, ci, al, col, d, ar, recs = inp
    kw = dict(us=us, cinv2ds=ci, alphas=al, colors=col)
    img = o.splat_features(H, W, col, out[1], out[3], out[4], **kw)
    assert torch.equal(bits(img), bits(out[0]))
    assert torch.equal(bits(o.splat_features(H, W, col, out[1], out[3], out[4], records=recs)), bits(out[0]))
    rgbd = o.splat_rgbd(H, W, us, ci, al, d, col, ar, records=recs)
    z = o.splat_features(H, W, d.reshape(-1, 1), out[1], out[3], out[4], records=recs)
    one = o.splat_features(H, W, torch.ones((N, 1), device=DEV), out[1], out[3], out[4], records=recs)
    assert torch.equal(bits(z[0]), bits(rgbd[5])) and torch.equal(bits(one[0]), bits(rgbd[6]))
    # backward: dL/dF = dL/dgamma with f = colours
    dl = t(upstream_gradient(W, H, 1) * (3.0 * W * H))
    m_col = o.splatB(H, W, us, ci, al, d, col, *out[1:5], dl, moments_only=True)
    g_col = o.splatB(H, W, us, ci, al, d, col, *out[1:5], dl)
    m_f, dfeat = o.splatB_features(H, W, col, out[1], out[2], out[3], out[4], dl, **kw)
    for k in range(6):
        a, b = m_col[:, k], m_f[:, k]
        assert float((a - b).abs().max()) <= 1e-5 * float(a.abs().max()), k
    ref = g_col[3].reshape(N, 3)
    assert float((dfeat - ref).abs().max()) <= 1e-5 * float(ref.abs().max())
    # chained after the colour rows: rows 0-5 double, rows 6-8 untouched
    m2, _ = o.splatB_features(H, W, col, out[1], out[2], out[3], out[4], dl, moments=m_col.clone(), **kw)
    assert torch.equal(m2[:, 6:], m_col[:, 6:])
    assert float((m2[:, :6] - 2 * m_col[:, :6]).abs().max()) <= 2e-5 * float(m_col[:, :6].abs().max())


# ---------------------------------------------------------------- 2. the oracle
@pytest.mark.parametrize("D", [1, 2, 3, 4, 5, 8, 16, 17, 32, 64])
def test_features_vs_oracle_every_width(D):
    N, W, H = 2000, 255, 131
    sc = scene_with_culls(N, W, H, 3, N + D)
    inp, out = frame(sc, W, H)
    check_features(H, W, inp, out, feats(N, D, D), seed=D)


@pytest.mark.parametrize("N,W,H,D", [(3000, 979, 546, 3), (3000, 979, 546, 17), (4001, 320, 200, 9),
                                     (40, 17, 9, 5), (8, 7, 5, 12)])
def test_features_vs_oracle_frame_sizes(N, W, H, D):
    sc = scene_with_culls(N, W, H, 3, N)
    inp, out = frame(sc, W, H)
    check_features(H, W, inp, out, feats(N, D, N), seed=N)


def test_whole_tile_entries_clamped_opacity_and_empty_tiles():
    """1..97-patch tiles (whole-tile and four-entry work items, chunk edges), opacities at and above the
    0.99 clamp (phase A's row-5 path) and most tiles of a wide frame empty (their zeros)"""
    rng = np.random.default_rng(9)
    gx, parts = 8, []
    tiles = [1, 2, 31, 32, 33, 63, 64, 65, 97, 34, 32, 40]
    for i, k in enumerate(tiles):
        p = gaussians_in_tile(i % gx, i // gx, k, rng, alpha=(0.02, 0.3) if k > 32 else (0.05, 0.9))
        if i in (9, 10):
            p[2][28:32] = (0.99, np.nextafter(np.float32(0.99), np.float32(1)), 1.0, 1.0)
        parts.append(p)
    us, ci, al, d, col, ar = op_inputs(parts)
    W, H = 16 * 40, 16 * 12
    out = ops().splat(H, W, us, ci, al, d, col, ar)
    f = feats(us.shape[0], 11, 3)
    fmap, ref, _ = check_features(H, W, (us, ci, al, col, d, ar, None), out, f, seed=3)
    lens = ref["ranges"][:, 1] - ref["ranges"][:, 0]
    empty = np.kron((lens == 0).reshape(H // 16, W // 16), np.ones((16, 16), bool))
    assert empty.mean() > 0.9 and not n(fmap)[:, empty].any()


def test_empty_scene_no_patches_and_misaligned_map():
    o = ops()
    W, H = 100, 70
    z2, z3 = torch.empty((0, 2), device=DEV), torch.empty((0, 3), device=DEV)
    out = o.splat(H, W, z2, z3, torch.empty(0, device=DEV), torch.empty(0, device=DEV), z3,
                  torch.empty((0, 2), dtype=torch.int32, device=DEV))
    f0 = torch.empty((0, 6), device=DEV)
    fmap = o.splat_features(H, W, f0, out[1], out[3], out[4])
    assert tuple(fmap.shape) == (6, H, W) and not bool(fmap.any())
    mom, dfeat = o.splatB_features(H, W, f0, out[1], out[2], out[3], out[4], torch.ones((6, H, W), device=DEV))
    assert tuple(mom.shape) == (0, 9) and tuple(dfeat.shape) == (0, 6)
    # every Gaussian behind the camera: P = 0, a zero map, zero gradients
    sc = synthetic_scene(500, W, H, sh_dim=3, seed=1)
    sc["pws"][:, 2] = -1.0
    inp, out = frame(sc, W, H)
    assert out[4].numel() == 0
    f = t(feats(500, 5, 1))
    fmap = o.splat_features(H, W, f, out[1], out[3], out[4])
    assert not bool(fmap.any())
    mom, dfeat = o.splatB_features(H, W, f, out[1], out[2], out[3], out[4], torch.ones((5, H, W), device=DEV))
    assert not bool(mom.any()) and not bool(dfeat.any())
    # a feature map that is not 16-byte aligned is refused by the entry point
    lib = o._L()
    sc = synthetic_scene(500, W, H, sh_dim=3, seed=2)
    inp, out = frame(sc, W, H)
    us, ci, al, col = inp[:4]
    buf = torch.empty(5 * H * W + 1, device=DEV)
    ws = torch.empty(lib.gsb_splat_features_workspace_bytes(500, H, W, out[4].numel()), dtype=torch.uint8, device=DEV)
    rc = lib.gsb_splat_features(H, W, 500, out[4].numel(), 5, us.data_ptr(), ci.data_ptr(), al.data_ptr(),
                                col.data_ptr(), f.data_ptr(), None, out[1].data_ptr(), out[3].data_ptr(),
                                out[4].data_ptr(), ws.data_ptr(), ws.numel(), buf.data_ptr() + 4,
                                torch.cuda.current_stream().cuda_stream)
    assert rc != 0 and b"misaligned feature_image" in lib.gsb_last_error()
    with pytest.raises(ValueError, match="records"):
        o.splat_features(H, W, f, out[1], out[3], out[4])  # neither records nor the attribute arrays


def test_capacity_path_overflow_fallback_and_record_sources():
    o = ops()
    N, W, H, D = 30000, 800, 600, 6
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=8)
    key = (torch.device(DEV).index or 0, H, W, N)
    o._CAPACITY.pop(key, None)
    inp, exact = frame(sc, W, H, capacity=True)
    us, ci, al, col, d, ar, recs = inp
    f = t(feats(N, D, 8))
    fm_exact = check_features(H, W, inp, exact, f, seed=8)[0]
    inp, cap = frame(sc, W, H, capacity=True)
    fm_cap = o.splat_features(H, W, f, cap[1], cap[3], cap[4], records=inp[6])
    assert torch.equal(bits(fm_cap), bits(fm_exact))
    o._CAPACITY[key] = (64, o._CAPACITY[key][1])  # far too few patch slots: redone the exact way
    before = o.CAPACITY_STATS["outgrown"]
    inp, over = frame(sc, W, H, capacity=True)
    assert o.CAPACITY_STATS["outgrown"] == before + 1
    fm_over = o.splat_features(H, W, f, over[1], over[3], over[4], records=inp[6])
    assert torch.equal(bits(fm_over), bits(fm_exact))
    # the records splat attached, and records packed again from the attribute arrays: the same bits
    us, ci, al, col, d, ar, recs = inp
    out = o.splat(H, W, us, ci, al, d, col, ar)
    kw = dict(us=us, cinv2ds=ci, alphas=al, colors=col)
    attached = o.splat_features(H, W, f, out[1], out[3], out[4], **kw)
    o.forget_records(out[4])
    repacked = o.splat_features(H, W, f, out[1], out[3], out[4], **kw)
    assert torch.equal(bits(attached), bits(fm_exact)) and torch.equal(bits(repacked), bits(fm_exact))


def test_features_at_an_odd_4_byte_offset():
    o = ops()
    N, W, H, D = 4001, 320, 200, 7
    sc = scene_with_culls(N, W, H, 3, 17)
    inp, out = frame(sc, W, H)
    f = feats(N, D, 17)
    flat = torch.empty(N * D + 1, device=DEV)
    flat[1:] = t(f).reshape(-1)
    odd = flat[1:].view(N, D)
    assert odd.data_ptr() % 16 == 4
    fm_odd, _, (m_odd, g_odd) = check_features(H, W, inp, out, odd, seed=17, records=inp[6])
    fm = o.splat_features(H, W, t(f), out[1], out[3], out[4], records=inp[6])
    assert torch.equal(bits(fm_odd), bits(fm))


# ---------------------------------------------------------------- 3. whole steps through the class
def run_features_class(sc, cam, f, F, dl, dF, need_image=True, need_map=True):
    from easygaussiansplatting_b200.gsfunction import GSFunctionFusedFeatures
    P = {k: t(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    al = t(sc["alphas"]).requires_grad_()
    us0 = torch.zeros((len(sc["pws"]), 2), device=DEV, requires_grad=True)
    fe = t(F).requires_grad_()
    outs = GSFunctionFusedFeatures.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us0, fe, cam,
                                         *(() if f is None else (t(f),)))
    loss = 0.0
    if need_image:
        loss = loss + (outs[0] * (t(dl) if dl is not None else 0.0)).sum()
    if need_map:
        loss = loss + (outs[1] * (t(dF) if dF is not None else 0.0)).sum()
    loss.backward()
    g = dict(pws=P["pws"].grad, shs=P["shs"].grad, scales=P["scales"].grad, rots=P["rots"].grad, alphas=al.grad,
             us=us0.grad, features=fe.grad)
    return outs, g


@pytest.mark.parametrize("aa,filt", [(False, False), (True, False), (False, True), (True, True)])
def test_class_step_vs_oracle(aa, filt):
    W, H, D = 640, 360, 5
    N = 20001
    sc, f, rows = matrix_scene(N, W, H, 4, seed=41 + 2 * aa + filt)
    f = f if filt else None
    rng = np.random.default_rng(3)
    F = rng.normal(size=(N, D)).astype(np.float32)
    dl = upstream_gradient(W, H, 4) * np.float32(3.0 * W * H)
    dF = (rng.normal(size=(D, H, W)) * 0.5).astype(np.float32)
    cam = _camera(sc, W, H, aa)
    outs, g = run_features_class(sc, cam, f, F, dl, dF)
    inp, ref = drawn_frame(sc, cam, f, False)
    assert torch.equal(bits(outs[0]), bits(ref[0]))
    fm = ops().splat_features(H, W, t(F), ref[1], ref[3], ref[4], records=None, us=t(inp["us"]),
                              cinv2ds=t(inp["ci"]), alphas=t(inp["alphas"]), colors=t(inp["col"]))
    assert torch.equal(bits(outs[1]), bits(fm))
    o = ofe.step_features(sc, ost.camera(sc, W, H), aa=aa, filt=f, features=F, dl=dl, dF=dF, drawn_inputs=inp)
    check_planes(outs, o, False)
    amb = o["ambiguous"] | o["thin_pixels"]
    e = np.abs(n(outs[1]).astype(np.float64) - o["features"]).max(0)
    assert e[~amb].max() <= 2e-4 * np.abs(F).max(), e[~amb].max()
    got = {k: n(v) for k, v in g.items()}
    check_grads(got, o["grads"], o["flagged"], o["band"], o["thin"], names=tuple(got))


# ---------------------------------------------------------------- 4. skip paths
def test_skip_paths_match_explicit_zero_gradients(monkeypatch):
    o = ops()
    W, H, D, N = 320, 240, 6, 8000
    # (no needle rows: the float atomics' summation order moves their gradients far more than 1e-5)
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=7)
    rng = np.random.default_rng(5)
    F = rng.normal(size=(N, D)).astype(np.float32)
    dl = upstream_gradient(W, H, 2) * np.float32(3.0 * W * H)
    dF = rng.normal(size=(D, H, W)).astype(np.float32)
    cam = _camera(sc, W, H, True)
    calls = {"splatB": 0, "splatB_features": 0}
    for name in calls:
        fn = getattr(o, name)

        def counted(*a, _fn=fn, _name=name, **k):
            calls[_name] += 1
            return _fn(*a, **k)
        monkeypatch.setattr(o, name, counted)

    def close(a, b, name):
        if a is None or b is None:
            assert (a is None or not bool(a.any())) and (b is None or not bool(b.any())), name
            return
        s = float(b.abs().max())
        assert float((a - b).abs().max()) <= 1e-5 * max(s, 1e-30), name

    # features only: the colour replay is skipped
    _, g_skip = run_features_class(sc, cam, None, F, None, dF, need_image=False)
    assert calls == {"splatB": 0, "splatB_features": 1}
    _, g_zero = run_features_class(sc, cam, None, F, np.zeros((3, H, W), np.float32), dF)
    assert calls == {"splatB": 1, "splatB_features": 2}
    for k in g_zero:
        close(g_skip[k], g_zero[k], k)
    assert bool(g_skip["features"].any()) and bool(g_skip["pws"].any())
    # colour only: the feature replay is skipped, and dL/dfeatures is None (or zero)
    _, g_skip = run_features_class(sc, cam, None, F, dl, None, need_map=False)
    assert calls == {"splatB": 2, "splatB_features": 2}
    _, g_zero = run_features_class(sc, cam, None, F, dl, np.zeros((D, H, W), np.float32))
    assert calls == {"splatB": 3, "splatB_features": 3}
    for k in g_zero:
        close(g_skip[k], g_zero[k], k)
    assert g_skip["features"] is None and not bool(g_zero["features"].any())
    # the multi-view exchange is refused
    from easygaussiansplatting_b200.gsfunction import GSFunctionFusedFeatures
    cam.grad_exchange = object()
    with pytest.raises(ValueError, match="grad_exchange"):
        GSFunctionFusedFeatures.apply(t(sc["pws"]), t(sc["shs"]), t(sc["alphas"]), t(sc["scales"]), t(sc["rots"]),
                                      torch.zeros((N, 2), device=DEV), t(F), cam)


# ---------------------------------------------------------------- 5. density
def _numpy_rebuild(cls, slots, counts, x, moment):
    K, C, S = counts
    out = np.zeros((K + C + S,) + x.shape[1:], x.dtype)
    for i in range(len(cls)):
        if cls[i] == 3:
            continue
        out[slots[i, 0]] = x[i]
        if cls[i] == 1:
            out[K + slots[i, 1]] = 0 if moment else x[i]
        elif cls[i] == 2:
            out[K + C + slots[i, 2]] = 0 if moment else x[i]
    return out


def _density_case(N, seed):
    """raw parameters + accumulators that prune, clone and split"""
    rng = np.random.default_rng(seed)
    sc = synthetic_scene(N, 64, 64, sh_dim=48, seed=seed)
    base = np.exp(rng.uniform(np.log(0.003), np.log(0.2), size=(N, 1)))  # sense size 1: clone <= 0.01 < split <= 0.1
    params = dict(pws=sc["pws"], low_shs=sc["shs"][:, :3], high_shs=sc["shs"][:, 3:],
                  alphas_raw=rng.normal(size=(N, 1)).astype(np.float32) * 3,
                  scales_raw=np.log(base * rng.uniform(0.8, 1.0, size=(N, 3))).astype(np.float32),
                  rots_raw=sc["rots"])
    acc = (rng.uniform(0, 2e-6, size=(N, 1))).astype(np.float32)
    cunt = rng.integers(1, 3, size=N).astype(np.int32)
    return params, acc, cunt


@pytest.mark.parametrize("D", [1, 5, 33])
def test_density_apply_rows_vs_numpy(D):
    from easygaussiansplatting_b200 import density
    N = 3001
    params, acc, cunt = _density_case(N, D)
    th = density.raw_thresholds(1.0)
    cls, slots, counts = density.plan(t(params["alphas_raw"]), t(params["scales_raw"]), t(acc), t(cunt, torch.int32),
                                      th)
    c = n(cls)
    assert all((c == k).any() for k in range(4)), np.bincount(c)
    x, m, v = (np.random.default_rng(D + i).normal(size=(N, D)).astype(np.float32) for i in range(3))
    dst, dm, dv = density.apply_rows(cls, slots, counts, t(x), t(m), t(v))
    for got, src, mom in ((dst, x, False), (dm, m, True), (dv, v, True)):
        assert np.array_equal(n(got), _numpy_rebuild(c, n(slots), counts, src, mom))
    only, none_m, none_v = density.apply_rows(cls, slots, counts, t(x))
    assert none_m is None and none_v is None and torch.equal(only, dst)


def test_density_controller_carries_features_with_adam():
    from easygaussiansplatting_b200.density import DensityController
    from easygaussiansplatting_b200.gau_io import adam_groups
    N, D = 4000, 16
    raw, acc, cunt = _density_case(N, 77)
    params = {k: t(v).requires_grad_() for k, v in raw.items()}
    params["features"] = t(feats(N, D, 9)).requires_grad_()
    groups = adam_groups({k: v for k, v in params.items() if k != "features"})
    opt = torch.optim.Adam(groups + [{"params": [params["features"]], "name": "features", "lr": 1e-2}], lr=1e-3)
    for p in params.values():  # one real Adam step: every group has state
        p.grad = torch.randn_like(p)
    opt.step()
    before = {k: n(p) for k, p in params.items()}
    m_before = {k: n(opt.state[p]["exp_avg"]) for k, p in params.items()}
    ctl = DensityController(1.0, verbose=False)
    ctl.grad_accum, ctl.cunt = t(acc), t(cunt, torch.int32)
    from easygaussiansplatting_b200 import density
    cls, slots, counts = density.plan(params["alphas_raw"].detach(), params["scales_raw"].detach(), ctl.grad_accum,
                                      ctl.cunt, ctl.th)
    c, sl = n(cls), n(slots)
    rep = ctl.update_gaussian_density(params, opt, extra=("features",))
    K, Cn, S = counts
    assert rep["pruned"] > 0 and rep["cloned"] > 0 and rep["splited"] > 0 and rep["total"] == K + Cn + S
    src = np.concatenate([np.flatnonzero(c != 3), np.flatnonzero(c == 1), np.flatnonzero(c == 2)])
    names = {g["name"]: g["params"][0] for g in opt.param_groups}
    for k, p in params.items():
        assert names[k] is p and p.shape[0] == K + Cn + S
        st = opt.state[p]
        assert st["exp_avg"].shape == p.shape and st["exp_avg_sq"].shape == p.shape
        assert np.array_equal(n(st["exp_avg"])[:K], m_before[k][src[:K]]), k  # survivors: aligned rows
        assert not n(st["exp_avg"])[K:].any(), k                               # new rows: zero moments
    assert np.array_equal(n(params["features"]), before["features"][src])    # every child copies its source
    assert np.array_equal(n(params["features"]), _numpy_rebuild(c, sl, counts, before["features"], False))
    assert np.array_equal(n(params["pws"])[:K + Cn], before["pws"][src[:K + Cn]])
    for p in params.values():  # the optimizer keeps stepping on the rebuilt tensors
        p.grad = torch.randn_like(p)
    opt.step()


# ---------------------------------------------------------------- 6. training
def test_feature_training_descends():
    """random features optimised toward per-Gaussian labels rendered from a hidden assignment: the
    geometry is frozen, only the feature map is used (no colour replay)"""
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFusedFeatures
    N, W, H, D = 5000, 160, 120, 4
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=21)
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]))
    frozen = [t(sc[k]) for k in ("pws", "shs")] + [t(sc["alphas"])] + [t(sc[k]) for k in ("scales", "rots")]
    us0 = torch.zeros((N, 2), device=DEV)
    labels = torch.nn.functional.one_hot(torch.from_numpy(np.random.default_rng(1).integers(0, D, N)), D).float().to(DEV)
    with torch.no_grad():
        target = GSFunctionFusedFeatures.apply(*frozen, us0, labels, cam)[1]
    fe = torch.nn.Parameter(torch.full((N, D), 1.0 / D, device=DEV) + 0.1 * torch.randn((N, D), device=DEV))
    opt = torch.optim.Adam([fe], lr=0.05)
    losses = []
    for _ in range(60):
        opt.zero_grad()
        fmap = GSFunctionFusedFeatures.apply(*frozen, us0, fe, cam)[1]
        loss = ((fmap - target) ** 2).mean()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert losses[-1] < 0.2 * losses[0], losses[::10]
