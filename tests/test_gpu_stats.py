"""Contribution statistics and the masked prune on the GPU (DESIGN 3.18).

1. `splat_stats` / `splat_surfel_stats` against the fp64 statistics oracles (oracle/stats_oracle.py)
   at the rasterizer edges: odd frames, empty tiles, whole-tile and dense tiles, the 0.99 clamp,
   N = 0, P = 0, the capacity path and its fallback, records given / attached / re-packed, outputs at
   an odd 4-byte offset.  hit_count exact and weight_max to 1e-4 off ambiguous Gaussians, weight_sum
   to 1e-4 of max|ref| (5e-3 on ambiguous ones), ambiguous Gaussians under 1 %.
2. Identities: sum weight_sum = sum of the alpha plane; weight_sum = splatB_features(ones)'s
   dL/dfeatures; two views accumulated = the sum of the single views (count and max bit-exact);
   at config 2 (1M Gaussians, 1920x1080, SH 3) too.
3. `density.prune` against torch's t[keep], with torch.optim.Adam and GaussianAdam; `lowest`;
   DensityController.prune.
4. Pruning the Gaussians no view composites changes no pixel of those views (colour and surfel)."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from oracle import stats_oracle as ost
from oracle import surfel_oracle as so
from easygaussiansplatting_b200.scene import ring_camera, synthetic_scene

from test_gpu_parity import DEV, gaussians_in_tile, n, op_inputs, scene_with_culls, t
from test_gpu_step_matrix import bits
from test_gpu_surfel import scene as surfel_scene

pytestmark = pytest.mark.gpu


def ops():
    from easygaussiansplatting_b200 import ops as o
    return o


def frame(sc, W, H, capacity=False):
    o = ops()
    al = t(sc["alphas"])
    us, ci, col, d, ar, recs = o.preprocess(*[t(sc[k]) for k in ("pws", "rots", "scales", "shs", "Rcw", "tcw", "twc")],
                                            sc["fx"], sc["fy"], sc["cx"], sc["cy"], W, H, alphas=al)
    out = o.splat(H, W, us, ci, al, d, col, ar, records=recs, capacity=capacity)
    return (us, ci, al, col, d, ar, recs), out


def check(got, ref):
    ws, wm, hc = (n(x) for x in got)
    amb = ref["ambiguous"]
    assert amb.mean() < 0.01, amb.mean()
    ok = ~amb
    assert np.array_equal(hc[ok], ref["hit_count"][ok])
    # weight_max to 1e-4 absolute (w <= 0.99: the image planes' tolerance against the fp64 oracle).  A
    # flat 1e-6 relative does not hold: a maximum taken far from the centre or behind many records
    # carries the fp32 exponent's and tau's roundings (up to ~2e-5 relative for surfels, measured
    # on the H100).  Maxima are compared bit for bit between GPU paths below.
    err_max = np.abs(wm.astype(np.float64) - ref["weight_max"])
    assert err_max[ok].max(initial=0) <= 1e-4, "weight_max err %.3e" % err_max[ok].max()
    s = max(np.abs(ref["weight_sum"]).max(initial=0), 1e-30)
    err = np.abs(ws.astype(np.float64) - ref["weight_sum"])
    assert err[ok].max(initial=0) <= 1e-4 * s, "weight_sum err %.3e" % (err[ok].max() / s)
    assert err.max(initial=0) <= 5e-3 * s
    assert wm.max(initial=0) <= np.float32(0.99)


def colour_case(H, W, inp, out, **kw):
    us, ci, al, col, d, ar, recs = inp
    ref_fwd = orc.splat(H, W, n(us), n(ci), n(al), n(d).copy(), n(col), n(ar).copy())
    assert np.array_equal(n(out[4]), ref_fwd["gsid"])
    ref = ost.splat_stats(H, W, n(us), n(ci), n(al), ref_fwd)
    got = ops().splat_stats(H, W, out[1], out[3], out[4], **kw)
    check(got, ref)
    return got, ref


# ---------------------------------------------------------------- 1. the oracle
@pytest.mark.parametrize("N,W,H", [(2000, 255, 131), (3000, 979, 546), (4001, 320, 200), (40, 17, 9), (8, 7, 5)])
def test_colour_stats_vs_oracle(N, W, H):
    sc = scene_with_culls(N, W, H, 3, N)
    inp, out = frame(sc, W, H)
    colour_case(H, W, inp, out, records=inp[6])


def test_whole_tile_dense_clamped_and_empty_tiles():
    rng = np.random.default_rng(9)
    gx, parts = 8, []
    for i, k in enumerate([1, 2, 31, 32, 33, 63, 64, 65, 97, 34, 32, 40]):
        p = gaussians_in_tile(i % gx, i // gx, k, rng, alpha=(0.02, 0.3) if k > 32 else (0.05, 0.9))
        if i in (9, 10):
            p[2][28:32] = (0.99, np.nextafter(np.float32(0.99), np.float32(1)), 1.0, 1.0)
        parts.append(p)
    us, ci, al, d, col, ar = op_inputs(parts)
    W, H = 16 * 40, 16 * 12
    out = ops().splat(H, W, us, ci, al, d, col, ar)
    got, ref = colour_case(H, W, (us, ci, al, col, d, ar, None), out, us=us, cinv2ds=ci, alphas=al, colors=col)
    assert n(got[1]).max() <= np.float32(0.99)
    lens = n(out[3])[:, 1] - n(out[3])[:, 0]
    assert (lens == 0).mean() > 0.9 and lens.max() >= 97


def test_empty_scene_and_no_patches():
    o = ops()
    W, H = 100, 70
    z2, z3 = torch.empty((0, 2), device=DEV), torch.empty((0, 3), device=DEV)
    out = o.splat(H, W, z2, z3, torch.empty(0, device=DEV), torch.empty(0, device=DEV), z3,
                  torch.empty((0, 2), dtype=torch.int32, device=DEV))
    ws, wm, hc = o.splat_stats(H, W, out[1], out[3], out[4], records=torch.empty((0, 12), device=DEV))
    assert ws.shape == (0,) and hc.dtype == torch.int64
    sc = synthetic_scene(500, W, H, sh_dim=3, seed=1)
    sc["pws"][:, 2] = -1.0  # every Gaussian behind the camera: P = 0
    inp, out = frame(sc, W, H)
    assert out[4].numel() == 0
    acc = (torch.full((500,), 2.0, device=DEV), torch.ones(500, device=DEV), torch.full((500,), 3, dtype=torch.int64,
                                                                                       device=DEV))
    got = o.splat_stats(H, W, out[1], out[3], out[4], records=inp[6], out=acc)
    assert got[0] is acc[0] and bool((acc[0] == 2).all() and (acc[1] == 1).all() and (acc[2] == 3).all())


def test_capacity_path_fallback_and_record_sources():
    o = ops()
    N, W, H = 30000, 800, 600
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=8)
    key = (torch.device(DEV).index or 0, H, W, N)
    o._CAPACITY.pop(key, None)
    inp, exact = frame(sc, W, H, capacity=True)
    want, _ = colour_case(H, W, inp, exact, records=inp[6])
    inp, cap = frame(sc, W, H, capacity=True)
    o._CAPACITY[key] = (64, o._CAPACITY[key][1])  # far too few patch slots: redone the exact way
    inp2, over = frame(sc, W, H, capacity=True)
    us, ci, al, col, d, ar, recs = inp2
    plain = o.splat(H, W, us, ci, al, d, col, ar)
    kw = dict(us=us, cinv2ds=ci, alphas=al, colors=col)
    attached = o.splat_stats(H, W, plain[1], plain[3], plain[4], **kw)
    o.forget_records(plain[4])
    repacked = o.splat_stats(H, W, plain[1], plain[3], plain[4], **kw)
    for got in (o.splat_stats(H, W, cap[1], cap[3], cap[4], records=inp[6]),
                o.splat_stats(H, W, over[1], over[3], over[4], records=recs), attached, repacked):
        assert torch.equal(got[1], want[1]) and torch.equal(got[2], want[2])  # exact: order-free
        assert float((got[0] - want[0]).abs().max()) <= 1e-5 * float(want[0].abs().max())


def test_outputs_at_an_odd_4_byte_offset():
    o = ops()
    N, W, H = 4001, 320, 200
    sc = scene_with_culls(N, W, H, 3, 17)
    inp, out = frame(sc, W, H)
    f = torch.zeros(2 * N + 1, device=DEV)
    h = torch.zeros(N + 1, dtype=torch.int64, device=DEV)
    odd = (f[1:N + 1], f[N + 1:], h[1:])
    assert odd[0].data_ptr() % 8 == 4 and odd[1].data_ptr() % 8 == 0 and odd[2].data_ptr() % 16 == 8
    o.splat_stats(H, W, out[1], out[3], out[4], records=inp[6], out=odd)
    ref = colour_case(H, W, inp, out, records=inp[6])[0]
    assert torch.equal(odd[1], ref[1]) and torch.equal(odd[2], ref[2]) and f[0] == 0 and h[0] == 0
    g = torch.zeros(N + 1, device=DEV)  # weight_max at an odd offset too
    o.splat_stats(H, W, out[1], out[3], out[4], records=inp[6], out=(odd[1].clone().zero_(), g[1:], h[1:].clone() * 0))
    assert torch.equal(g[1:], ref[1])


def surfel_frame(sc):
    o = ops()
    P = {k: t(sc[k]) for k in ("pws", "rots", "scales", "shs", "alphas", "Rcw", "tcw", "twc")}
    cam = (sc["fx"], sc["fy"], sc["cx"], sc["cy"], sc["W"], sc["H"])
    us, depths, areas, colors, recs = o.surfel_preprocess(P["pws"], P["rots"], P["scales"], P["shs"], P["alphas"],
                                                          P["Rcw"], P["tcw"], P["twc"], *cam)
    out = o.splat_surfel(sc["H"], sc["W"], us, depths, areas, recs)
    return (us, depths, areas, recs), out


@pytest.mark.parametrize("N,W,H,spread", [(3, 40, 24, 0.3), (60, 72, 40, 1.1), (400, 90, 60, 1.2),
                                          (1500, 64, 48, 1.0), (5000, 161, 97, 1.0)])
def test_surfel_stats_vs_oracle(N, W, H, spread):
    sc = surfel_scene(N, W, H, k=1, seed=N, spread=spread)
    sc["alphas"][: max(1, N // 50)] = 1.0  # clamped near their centres
    (us, depths, areas, recs), out = surfel_frame(sc)
    got = ops().splat_surfel_stats(H, W, recs, out[1], out[3], out[4])
    pre = so.preprocess(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                        sc["fy"], sc["cx"], sc["cy"])
    bins = so.orc.bin(H, W, n(us), n(depths).copy(), n(areas).copy())
    ref = ost.surfel_stats(H, W, pre, sc["alphas"], bins)
    check(got, ref)
    # the identity with the frame's alpha plane
    assert abs(float(got[0].double().sum()) - float(out[6].double().sum())) <= 1e-5 * float(out[6].double().sum())


def test_surfel_empty_frame():
    sc = surfel_scene(0, 33, 17)
    (_, _, _, recs), out = surfel_frame(sc)
    ws, wm, hc = ops().splat_surfel_stats(17, 33, recs, out[1], out[3], out[4])
    assert ws.shape == (0,)


# ---------------------------------------------------------------- 2. identities
@pytest.mark.parametrize("N,W,H", [(20000, 640, 480), (3000, 979, 546), (1_000_000, 1920, 1080)])
def test_identities(N, W, H):
    o = ops()
    sc = synthetic_scene(N, W, H, sh_dim=48, seed=N)
    inp, out = frame(sc, W, H)
    us, ci, al, col, d, ar, recs = inp
    ws, wm, hc = o.splat_stats(H, W, out[1], out[3], out[4], records=recs)
    rgbd = o.splat_rgbd(H, W, us, ci, al, d, col, ar, records=recs)
    A = float(rgbd[6].double().sum())
    assert abs(float(ws.double().sum()) - A) <= 1e-5 * A
    ones = torch.ones((N, 1), device=DEV)
    _, df = o.splatB_features(H, W, ones, out[1], out[2], out[3], out[4], torch.ones((1, H, W), device=DEV),
                              records=recs)
    assert float((df[:, 0] - ws).abs().max()) <= 1e-5 * float(ws.abs().max())
    assert int(hc.sum()) > 0 and float(wm.max()) <= 0.99
    # two views accumulated = the sum of the single views
    sc2 = dict(sc)
    sc2["Rcw"], sc2["tcw"], sc2["twc"] = ring_camera(1, 8)
    inp2, out2 = frame(sc2, W, H)
    v2 = o.splat_stats(H, W, out2[1], out2[3], out2[4], records=inp2[6])
    acc = o.splat_stats(H, W, out[1], out[3], out[4], records=recs)
    o.splat_stats(H, W, out2[1], out2[3], out2[4], records=inp2[6], out=acc)
    assert torch.equal(acc[2], hc + v2[2]) and torch.equal(acc[1], torch.maximum(wm, v2[1]))
    assert float((acc[0] - (ws + v2[0])).abs().max()) <= 1e-5 * float(acc[0].abs().max())


# ---------------------------------------------------------------- 3. prune
def _params(N, seed, optimizer, state):
    from easygaussiansplatting_b200.gau_io import adam_groups
    from easygaussiansplatting_b200.optim import GaussianAdam
    rng = np.random.default_rng(seed)
    widths = dict(pws=3, low_shs=3, high_shs=45, alphas_raw=1, scales_raw=3, rots_raw=4)
    params = {k: t(rng.normal(size=(N, w)).astype(np.float32)).requires_grad_() for k, w in widths.items()}
    params["features"] = t(rng.normal(size=(N, 5)).astype(np.float32)).requires_grad_()
    groups = adam_groups({k: v for k, v in params.items() if k != "features"})
    groups = groups + [{"params": [params["features"]], "name": "features", "lr": 1e-2}]
    opt = (torch.optim.Adam if optimizer == "adam" else GaussianAdam)(groups, lr=1e-3)
    if state:
        for p in params.values():
            p.grad = torch.randn_like(p)
        opt.step()
    return params, opt


@pytest.mark.parametrize("optimizer", ["adam", "gaussian_adam"])
@pytest.mark.parametrize("state", [True, False])
def test_prune_matches_boolean_indexing(optimizer, state):
    from easygaussiansplatting_b200.density import prune
    N = 5000
    for kind in ("random", "all", "none"):
        params, opt = _params(N, 3, optimizer, state)
        keep = {"random": torch.rand(N, device=DEV) < 0.6, "all": torch.ones(N, dtype=torch.bool, device=DEV),
                "none": torch.zeros(N, dtype=torch.bool, device=DEV)}[kind]
        before = {k: p.detach().clone() for k, p in params.items()}
        mom = {k: (opt.state[p]["exp_avg"].clone(), opt.state[p]["exp_avg_sq"].clone(), opt.state[p]["step"])
               for k, p in params.items()} if state else None
        rep = prune(params, opt, keep, extra=("features",), verbose=False)
        K = int(keep.sum())
        assert rep == dict(pruned=N - K, total=K)
        names = {g["name"]: g["params"][0] for g in opt.param_groups}
        for k, p in params.items():
            assert names[k] is p and p.shape[0] == K
            assert torch.equal(bits(p.detach()), bits(before[k][keep])), k
            if state:
                st = opt.state[p]
                assert torch.equal(bits(st["exp_avg"]), bits(mom[k][0][keep])), k
                assert torch.equal(bits(st["exp_avg_sq"]), bits(mom[k][1][keep])), k
                assert st["step"] is mom[k][2] or torch.equal(torch.as_tensor(st["step"]), torch.as_tensor(mom[k][2]))
            else:
                assert p not in opt.state
        if kind == "none":  # N = 0: a following forward works
            o = ops()
            z = torch.zeros((0, 3), device=DEV)
            pre = o.preprocess(params["pws"].detach(), params["rots_raw"].detach(), z, torch.zeros((0, 3), device=DEV),
                               t(np.eye(3)), t(np.zeros(3)), t(np.zeros(3)), 100.0, 100.0, 32.0, 24.0, 64, 48)
            img = o.splat(48, 64, pre[0], pre[1], torch.zeros(0, device=DEV), pre[3], pre[2], pre[4])[0]
            assert not bool(img.any())
        for p in params.values():  # the optimizer keeps stepping on the pruned tensors
            p.grad = torch.randn_like(p)
        opt.step()


def test_density_controller_prune_resets_its_statistics():
    from easygaussiansplatting_b200.density import DensityController
    N = 3000
    params, opt = _params(N, 5, "adam", True)
    ctl = DensityController(1.0, verbose=False)
    ctl.update_density_info(torch.randn((N, 2), device=DEV), torch.ones(N, dtype=torch.bool, device=DEV))
    assert ctl.cunt is not None
    keep = torch.rand(N, device=DEV) < 0.5
    rep = ctl.prune(params, opt, keep, extra=("features",))
    assert ctl.cunt is None and ctl.grad_accum is None and rep["total"] == int(keep.sum())
    with pytest.raises(RuntimeError):
        ctl.update_gaussian_density(params, opt, extra=("features",))


def test_lowest_on_the_device():
    from easygaussiansplatting_b200.density import lowest
    s = torch.tensor([3.0, 1.0, 1.0, 2.0, 1.0, 0.5], device=DEV)
    assert lowest(s, 0.5).tolist() == [True, False, False, True, True, False]
    r = torch.randint(0, 5, (100001,), device=DEV).float()
    keep = lowest(r, 0.3)
    assert int((~keep).sum()) == 30000
    order = np.lexsort((np.arange(r.numel()), n(r)))
    want = np.ones(r.numel(), bool)
    want[order[:30000]] = False
    assert np.array_equal(n(keep), want)


# ---------------------------------------------------------------- 4. pruning dead Gaussians changes no pixel
def _cams(sc, n_views, W, H):
    from easygaussiansplatting_b200.gsfunction import Camera
    cams = []
    for v in range(n_views):
        Rcw, tcw, twc = ring_camera(v, n_views)
        cams.append(Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(Rcw), t(tcw), t(twc)))
    return cams


def test_pruning_dead_gaussians_changes_no_pixel():
    from easygaussiansplatting_b200.gsfunction import GSFunctionFusedRGBD, contribution_stats
    N, W, H = 60000, 480, 320
    sc = synthetic_scene(N, W, H, sh_dim=48, seed=21)
    cams = _cams(sc, 6, W, H)
    P = dict(pws=t(sc["pws"]), shs=t(sc["shs"]), alphas=t(sc["alphas"][:, None]), scales=t(sc["scales"]),
             rots=t(sc["rots"]))

    def render(P):
        with torch.no_grad():
            return [GSFunctionFusedRGBD.apply(P["pws"], P["shs"], P["alphas"], P["scales"], P["rots"],
                                              torch.zeros((P["pws"].shape[0], 2), device=DEV), c)[:3] for c in cams]

    st = contribution_stats(P["pws"], P["shs"], P["alphas"], P["scales"], P["rots"], cams)
    keep = st["hit_count"] > 0
    assert 0 < int((~keep).sum()) < N
    assert bool(((st["views"] > 0) == keep).all()) and int(st["views"].max()) <= len(cams)
    before = render(P)
    after = render({k: v[keep] for k, v in P.items()})
    for a, b in zip(before, after):
        for x, y in zip(a, b):
            assert torch.equal(bits(x), bits(y))


def test_pruning_dead_surfels_changes_no_pixel():
    from easygaussiansplatting_b200.gsfunction import GSFunctionSurfel, contribution_stats
    N, W, H = 20000, 320, 200
    sc = surfel_scene(N, W, H, k=16, seed=22)
    sc["width"], sc["height"] = W, H
    cams = _cams(sc, 4, W, H)
    P = dict(pws=t(sc["pws"]), shs=t(sc["shs"]), alphas=t(sc["alphas"][:, None]), scales=t(sc["scales"]),
             rots=t(sc["rots"]))

    def render(P):
        with torch.no_grad():
            return [GSFunctionSurfel.apply(P["pws"], P["shs"], P["alphas"], P["scales"], P["rots"],
                                           torch.zeros((P["pws"].shape[0], 2), device=DEV), c)[:4] for c in cams]

    st = contribution_stats(P["pws"], P["shs"], P["alphas"], P["scales"], P["rots"], cams, surfel=True)
    keep = st["hit_count"] > 0
    assert 0 < int((~keep).sum()) < N
    before = render(P)
    after = render({k: v[keep] for k, v in P.items()})
    for a, b in zip(before, after):
        for x, y in zip(a, b):
            assert torch.equal(bits(x), bits(y))
