"""2DGS geometry terms on the H100 (k_draw_2dgs, k_draw_2dgs_bwd, splat_surfel_geometry,
GSFunctionSurfelGeometry) against the fp64 model of tests/surfel_geometry_oracle.py, binned
independently, and against the surfel path they extend.

1. The surfel planes of the geometry frame equal splat_surfel's bit for bit (one walk).
2. distortion, moments, median_depth and median_contrib against the model on the kernels' own
   records, per pixel: |distortion - model| <= 1e-4 cond + 2^-20 A^2 with cond = sum w (m^2 A + D2 +
   2 m D) = 2 (A D2 + D^2) the pixel's fp64 conditioning (A^2: the fp32 rounding of m near `near`).
3. Rows against the model per entry (within 1e-4 of the entry's absolute sum), and the parameter
   gradients of k_surfel_bwd on those rows: dL/ddistortion alone, dL/dmedian alone, all six planes.
4. With no geometry gradient splatB_surfel_geometry runs k_draw_surfel_bwd, not k_draw_2dgs_bwd, and
   its rows are splatB_surfel's up to the order of their float atomics (as are k_draw_2dgs_bwd's with
   explicit zero geometry gradients); the capacity path equals the exact path bit for bit.
5. Training: the distortion of two parallel disks falls at every step; a run with DensityController
   and GaussianAdam stays finite."""
import numpy as np
import pytest
import torch

from oracle import surfel_oracle as so
import surfel_geometry_oracle as sg
from test_gpu_surfel_edges import T, cam_args, gpu_preprocess, n, ops, params, pre_of, record_pre, rows_bound
from test_surfel_edge_scenes_cpu import fronto, place, random_scene, stack_scene

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def geo_frame(sc, near=0.2, far=100.0, capacity=False):
    g = gpu_preprocess(sc)
    out = ops().splat_surfel_geometry(sc["H"], sc["W"], g[0], g[1], g[2], g[4], near, far, capacity=capacity)
    return g, out


def check_geometry(sc, near=0.2, far=100.0):
    """the geometry planes against the model on the kernels' records -> dict for the backward checks"""
    H, W = sc["H"], sc["W"]
    g, out = geo_frame(sc, near, far)
    recs = n(g[4])
    pre = pre_of(sc)
    bins = so.bin_f32(H, W, pre)
    ranges, gsid = n(out[3]), n(out[4])
    assert np.array_equal(ranges, bins[1]) and np.array_equal(gsid, bins[2])
    rp = record_pre(pre, recs)
    fwd = sg.render_geometry(H, W, rp, sc["alphas"], bins, near, far)
    ok = ~fwd["ambiguous"]
    assert ok.mean() > 0.5
    dist, med, mom, medc = (n(x) for x in out[8:])
    A, D, D2 = fwd["alpha"], fwd["moments"][0], fwd["moments"][1]
    cond = 2 * (A * D2 + D * D)
    tol = 1e-4 * cond + 2.0 ** -20 * A * A + 1e-30
    r = np.abs(dist - fwd["distortion"]) / tol
    assert r[ok].max(initial=0) <= 1.0, float(r[ok].max())
    for k in range(2):
        e = np.abs(mom[k] - fwd["moments"][k]) / (1e-4 * fwd["moments"][k] + 2.0 ** -20 * A + 1e-30)
        assert e[ok].max(initial=0) <= 1.0, (k, float(e[ok].max()))
    assert (medc == fwd["median_contrib"])[ok].all()
    assert np.abs(med - fwd["median_depth"])[ok].max(initial=0) <= 1e-4 * max(1.0, np.abs(fwd["median_depth"]).max())
    assert not med[medc == 0].any()
    # empty tiles: every geometry plane is 0
    live = np.repeat(np.repeat((bins[1][:, 1] > bins[1][:, 0]).reshape((H + 15) // 16, (W + 15) // 16), 16, 0),
                     16, 1)[:H, :W]
    assert not dist[~live].any() and not mom[:, ~live].any() and not med[~live].any() and not medc[~live].any()
    return dict(g=g, out=out, pre=pre, rp=rp, bins=bins, fwd=fwd, ok=ok)


def test_geometry_frame_planes_equal_splat_surfel():
    for cam, N, W, H, seed in (("posed_a", 700, 203, 121, 1), ("posed_b", 3000, 333, 197, 2)):
        sc = random_scene(N, W, H, 4, cam=cam, seed=seed, spread=1.1)
        g = gpu_preprocess(sc)
        ref = ops().splat_surfel(H, W, g[0], g[1], g[2], g[4])
        _, out = geo_frame(sc)
        for a, b in zip(ref, out[:8]):
            assert torch.equal(a, b)


@pytest.mark.parametrize("cam,N,W,H,k3", [("identity", 3, 45, 29, 1), ("posed_a", 700, 203, 121, 4),
                                          ("posed_b", 4000, 333, 197, 16), ("posed_a", 20000, 517, 301, 1)])
def test_geometry_planes_match_the_model(cam, N, W, H, k3):
    sc = random_scene(N, W, H, k3, cam=cam, seed=N + k3, spread=1.1, z=(1.0, 6.0) if N <= 4000 else (2.0, 6.0))
    res = check_geometry(sc)
    if N >= 700:
        assert (n(res["out"][8]) > 0).mean() > 0.2
    if N <= 700:
        check_geometry(sc, near=1.5, far=20.0)   # hits on both sides of near


def test_geometry_planes_on_whole_tile_entries_and_stacks():
    sc, _ = stack_scene()
    check_geometry(sc, near=2.9, far=50.0)


def test_geometry_planes_at_4k():
    sc = random_scene(400, 3840, 2160, 1, cam="posed_b", seed=4, spread=1.0, size=(0.005, 0.03))
    check_geometry(sc)


def check_rows(sc, res, dl, near, far):
    o = ops()
    H, W = sc["H"], sc["W"]
    g, out = res["g"], res["out"]
    t = [None if d is None else T(d.astype(np.float32)) for d in dl]
    rows = o.splatB_surfel_geometry(H, W, g[4], out[1], out[2], out[3], out[4], out[6], out[10], out[11], *t,
                                    near=near, far=far)
    want, ab = sg.render_backward_geometry(H, W, res["rp"], sc["alphas"], res["bins"], res["fwd"], *dl, near=near,
                                           far=far, abs_rows=True)
    rows_n = n(rows)
    rows_bound(rows_n, want, ab, "rows")
    assert np.abs(rows_n).max() > 0
    P = params(sc)
    gr = o.surfel_preprocessB(P["pws"], P["rots"], P["scales"], P["shs"], P["Rcw"], P["tcw"], P["twc"], *cam_args(sc),
                              rows)
    ref = so.preprocess_backward(res["pre"], rows_n.astype(np.float64))
    names = ("pws", "shs", "alphas", "scales", "rots", "us")
    N = len(sc["pws"])
    got = np.concatenate([n(x).reshape(N, -1) for x in gr], 1).astype(np.float64)
    exp = np.concatenate([ref[k].reshape(N, -1) for k in names], 1)
    K = res["pre"]["K"]
    norm = np.maximum(np.linalg.norm(exp, axis=1), 1e-3 * np.abs(K).sum() * np.linalg.norm(rows_n, axis=1))
    assert (np.abs(got - exp).max(axis=1) <= 1e-4 * norm + 1e-30).all()
    return rows


@pytest.mark.parametrize("planes", ["distortion", "median", "all"])
@pytest.mark.parametrize("cam,N,W,H,k3,near", [("posed_a", 400, 141, 93, 4, 0.2), ("posed_b", 1500, 203, 121, 9, 1.5)])
def test_geometry_rows_match_the_model(cam, N, W, H, k3, near, planes):
    far = 40.0
    sc = random_scene(N, W, H, k3, cam=cam, seed=N + 5, spread=1.1, z=(1.0, 6.0))
    res = check_geometry(sc, near, far)
    rng = np.random.default_rng(N)
    ok = res["ok"]
    full = [rng.normal(size=(3, H, W)), rng.normal(size=(H, W)), rng.normal(size=(H, W)), rng.normal(size=(3, H, W)),
            rng.normal(size=(H, W)) * 10, rng.normal(size=(H, W))]
    use = {"distortion": (4,), "median": (5,), "all": range(6)}[planes]
    dl = [np.where(ok, a, 0.0) if i in use else None for i, a in enumerate(full)]
    check_rows(sc, res, dl, near, far)


def test_rows_without_geometry_gradients_are_splatB_surfels():
    from easygaussiansplatting_b200 import _lib
    lib = _lib.load()
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    k_s, k_g = names.index("draw_surfel_backward"), names.index("draw_2dgs_backward")
    o = ops()
    sc = random_scene(900, 160, 96, 4, cam="posed_a", seed=9, spread=1.1)
    g, out = geo_frame(sc)
    rng = np.random.default_rng(1)
    dl = [T(rng.normal(size=s).astype(np.float32)) for s in ((3, 96, 160), (96, 160), (96, 160), (3, 96, 160))]
    ref = o.splatB_surfel(96, 160, g[4], out[1], out[2], out[3], out[4], *dl)
    s0, g0 = lib.gsb_profile_launches(k_s), lib.gsb_profile_launches(k_g)
    # the rows are float atomics: two runs of one kernel agree up to the order of their additions
    same = lambda r: torch.allclose(r, ref, rtol=1e-4, atol=1e-6 * float(ref.abs().max()))
    rows = o.splatB_surfel_geometry(96, 160, g[4], out[1], out[2], out[3], out[4], out[6], out[10], out[11], *dl)
    torch.cuda.synchronize()
    assert same(rows)
    assert lib.gsb_profile_launches(k_s) == s0 + 1 and lib.gsb_profile_launches(k_g) == g0
    z = torch.zeros((96, 160), device=DEV)
    rows = o.splatB_surfel_geometry(96, 160, g[4], out[1], out[2], out[3], out[4], out[6], out[10], out[11], *dl, z, z)
    torch.cuda.synchronize()
    assert lib.gsb_profile_launches(k_g) == g0 + 1
    assert same(rows)   # a zero geometry gradient adds exact zeros


def test_geometry_capacity_path_matches_exact_path():
    sc = random_scene(2000, 203, 121, 4, cam="posed_b", seed=12, spread=1.1)
    ops()._CAPACITY.clear()
    _, exact = geo_frame(sc, 0.3, 30.0, capacity=True)   # learns the bounds
    _, cap = geo_frame(sc, 0.3, 30.0, capacity=True)
    assert ops().CAPACITY_STATS["capacity_frames"] > 0
    for a, b in zip(exact, cap):
        assert torch.equal(a, b)


def test_gsfunction_geometry_autograd_and_refusals():
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionSurfel, GSFunctionSurfelGeometry
    sc = random_scene(500, 96, 64, 4, cam="posed_a", seed=3, spread=1.1)
    cam = Camera(96, 64, sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(sc["Rcw"]), T(sc["tcw"]), T(sc["twc"]))
    P = {k: T(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    al = T(sc["alphas"][:, None]).requires_grad_()
    us = torch.zeros((500, 2), device=DEV, requires_grad=True)
    outs = GSFunctionSurfelGeometry.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us, cam)
    ref = GSFunctionSurfel.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us, cam)
    for a, b in zip(outs[:4], ref[:4]):
        assert torch.equal(a, b)
    assert torch.equal(outs[6], ref[4])
    # no gradient on the geometry planes: GSFunctionSurfel's gradients, bit for bit
    leaves = [P["pws"], P["shs"], al, P["scales"], P["rots"], us]
    g1 = torch.autograd.grad(outs[0].sum() + outs[2].sum(), leaves)
    g2 = torch.autograd.grad(ref[0].sum() + ref[2].sum(), leaves)
    for a, b in zip(g1, g2):   # (float atomics: equal up to their order)
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-6 * float(b.abs().max()))
    outs = GSFunctionSurfelGeometry.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us, cam, 0.5, 20.0)
    g3 = torch.autograd.grad(outs[4].sum() + outs[5].mean(), leaves)
    assert all(torch.isfinite(x).all() for x in g3) and g3[0].abs().max() > 0
    for bad in (dict(near=0.0), dict(near=2.0, far=1.0), dict(far=float("inf")), dict(near=torch.ones(1)),
                dict(near=torch.zeros((500, 1)), far=None)):
        with pytest.raises(ValueError):
            GSFunctionSurfelGeometry.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us, cam,
                                           bad.get("near", 0.2), bad.get("far", 100.0))
    cam.antialiased = True
    with pytest.raises(ValueError, match="GSFunctionSurfelGeometry"):
        GSFunctionSurfelGeometry.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us, cam)
    cam.antialiased = False
    cam.grad_exchange = object()
    with pytest.raises(ValueError, match="GSFunctionSurfelGeometry"):
        GSFunctionSurfelGeometry.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us, cam)


def test_distortion_of_two_parallel_disks_falls():
    """two overlapping fronto-parallel disks at z 2.0 and 2.6: gradient descent on the positions at a
    fixed lr lowers the summed distortion at every step"""
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionSurfelGeometry
    W, H = 96, 80
    sc = place(np.array([[0.02, -0.01, 2.0], [-0.03, 0.02, 2.6]]), fronto(2), np.array([[0.5, 0.45, 0.0]] * 2),
               np.zeros((2, 3)), np.array([0.6, 0.7]), "posed_a", W, H)
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(sc["Rcw"]), T(sc["tcw"]), T(sc["twc"]))
    pws = T(sc["pws"]).requires_grad_()
    fixed = [T(sc[k]) for k in ("shs", "alphas", "scales", "rots")]
    losses = []
    for _ in range(25):
        us = torch.zeros((2, 2), device=DEV, requires_grad=True)
        outs = GSFunctionSurfelGeometry.apply(pws, fixed[0], fixed[1][:, None], fixed[2], fixed[3], us, cam)
        loss = outs[4].sum()
        (gp,) = torch.autograd.grad(loss, [pws])
        with torch.no_grad():
            pws -= 1e-2 * gp
        losses.append(float(loss.detach()))
    assert losses[0] > 0
    assert all(b < a for a, b in zip(losses, losses[1:])), losses
    assert losses[-1] < 0.9 * losses[0], losses


def test_geometry_training_with_density_control_and_gaussian_adam():
    from easygaussiansplatting_b200.density import DensityController
    from easygaussiansplatting_b200.gau_io import adam_groups
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionSurfelGeometry
    from easygaussiansplatting_b200.loss import depth_to_normal
    from easygaussiansplatting_b200.optim import GaussianAdam
    from easygaussiansplatting_b200.scene import synthetic_scene
    N, W, H = 3000, 128, 96
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=7)
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(sc["Rcw"]), T(sc["tcw"]), T(sc["twc"]))
    with torch.no_grad():
        target = GSFunctionSurfelGeometry.apply(T(sc["pws"]), T(sc["shs"]), T(sc["alphas"][:, None]),
                                                T(sc["scales"]), T(sc["rots"]), torch.zeros((N, 2), device=DEV), cam)[0]
    rng = np.random.default_rng(8)
    raw = dict(pws=sc["pws"] + rng.normal(size=(N, 3)).astype(np.float32) * 0.02,
               low_shs=np.zeros((N, 3), np.float32), high_shs=np.zeros((N, 45), np.float32),
               alphas_raw=np.log(sc["alphas"] / (1 - sc["alphas"])).astype(np.float32).reshape(N, 1),
               scales_raw=np.log(np.maximum(sc["scales"], 1e-3)).astype(np.float32), rots_raw=sc["rots"])
    P = {k: torch.nn.Parameter(T(np.ascontiguousarray(v, dtype=np.float32))) for k, v in raw.items()}
    opt = GaussianAdam(adam_groups(P), lr=1e-3)
    ctl = DensityController(sense_size=5.0, verbose=False)
    for step in range(40):
        opt.zero_grad()
        us = torch.zeros((P["pws"].shape[0], 2), device=DEV, requires_grad=True)
        img, depth, alpha, normal, dist, med, mask = GSFunctionSurfelGeometry.apply(
            P["pws"], torch.cat([P["low_shs"], P["high_shs"][:, :9]], 1), torch.sigmoid(P["alphas_raw"]),
            torch.exp(P["scales_raw"]), torch.nn.functional.normalize(P["rots_raw"], dim=1), us, cam)
        ln = (1 - (normal * depth_to_normal(med, cam) * alpha.detach()).sum(0)).mean()
        loss = (img - target).abs().mean() + 100.0 * dist.mean() + 0.05 * ln
        loss.backward()
        assert torch.isfinite(loss)
        ctl.update_density_info(us.grad, mask)
        opt.step()
        if step == 19:
            ctl.update_gaussian_density(P, opt)
        assert all(torch.isfinite(p).all() for p in P.values())
