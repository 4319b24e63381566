"""GPU checks of the Mip-Splatting 3D smoothing filter: ops.filter3d against the fp64 oracle
(oracle/filter3d_oracle.py) over N, camera counts around the shared-memory chunk, unseen rows and
frames, cameras with different fx, determinism and offset views; ops.filter3d_apply /
filter3d_backward against the oracle in and out of place; the four fused classes with and without
antialiasing, GraphedFusedStep, MultiViewStep and the gradient exchange with a filter; a zero filter
reproducing today's step; and gau_io.bake_filter3d."""
import numpy as np
import pytest
import torch

from oracle import filter3d_oracle as of3
from easygaussiansplatting_b200 import _lib
from easygaussiansplatting_b200.scene import ring_camera, synthetic_scene, upstream_gradient

from test_filter3d_cpu import box_points, edge_rows, ring_table

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CHUNK = 64  # ops.FILTER3D_CHUNK, asserted below


def t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).to(DEV)


def n(x):
    return x.detach().cpu().numpy()


def bits(x):
    return x.detach().contiguous().view(torch.int32)


def test_chunk_constant():
    from easygaussiansplatting_b200 import ops
    assert ops.FILTER3D_CHUNK == CHUNK


CASES = [(N, C) for N in (1, 127, 129, 20001) for C in (1, 7, CHUNK - 1, CHUNK, CHUNK + 1, 2 * CHUNK + 1)] + \
    [(2001, 3000), (1048577, 7), (1048577, CHUNK + 1)]


@pytest.mark.parametrize("N,C", CASES)
def test_filter3d_vs_oracle(N, C):
    """d_i bit for bit on unflagged rows (variance = fmax^2, fmax = 512: the filter is d itself), the
    value at variance 0.2 to 1e-6, two calls bit-identical, an offset pws view the same bits"""
    from easygaussiansplatting_b200 import ops
    pws, far = box_points(N, seed=N + C)
    table = ring_table(C, seed=N * 7 + C)
    table[C // 2, 12] = 512.0  # the largest fx, a power of two; fx differs between cameras
    ref = of3.filter3d(pws, table)
    ok = ~ref["flagged"]
    # a decision within 1e-6 of a bound: about 1.3e-6 of the (row, camera) pairs on these rings
    assert ref["flagged"].sum() <= max(3, 4 * N * C // 10 ** 6), ref["flagged"].sum()
    P, T = t(pws), t(table)
    d = ops.filter3d(P, T, variance=512.0 ** 2)
    assert np.array_equal(n(d)[ok], ref["d"][ok].astype(np.float32))
    f1 = ops.filter3d(P, T)
    f2 = ops.filter3d(P, T)
    assert torch.equal(bits(f1), bits(f2))
    got = n(f1).astype(np.float64)
    assert np.all(np.abs(got - ref["filter"])[ok] <= 1e-6 * ref["filter"][ok])
    if N > 1:
        assert not ref["seen"][far].any() and (got[far] == got.max()).all() if far.any() else True
    buf = torch.empty(3 * N + 1, device=DEV)
    buf[1:] = P.reshape(-1)
    assert torch.equal(bits(ops.filter3d(buf[1:].view(N, 3), T)), bits(f1))


def test_filter3d_nothing_seen_and_no_cameras():
    from easygaussiansplatting_b200 import ops
    pws = t(np.random.default_rng(1).uniform(-1, 1, (5000, 3)) + [0, 500, 0])
    assert not ops.filter3d(pws, t(ring_table(9, seed=3))).any()
    assert not ops.filter3d(pws, torch.zeros((0, 20), device=DEV)).any()
    assert ops.filter3d(pws[:0], t(ring_table(3, seed=3))).numel() == 0


def test_filter3d_without_a_positive_fx():
    """f_max is the largest positive fx: a table whose fx are all <= 0 gives zeros (not d / 0), and a
    camera with fx <= 0 among others only drops out of the maximum (the table is not checked)"""
    from easygaussiansplatting_b200 import ops
    pws, _ = box_points(20001, seed=11)
    table = ring_table(9, seed=12)
    bad = table.copy()
    bad[:, 12] = -np.abs(bad[:, 12])
    bad[0, 12] = 0.0
    assert not ops.filter3d(t(pws), t(bad)).any()
    mixed = table.copy()
    mixed[3, 12] = -1000.0
    ref = of3.filter3d(pws, mixed)
    assert ref["fmax"] == float(np.max(table[np.arange(9) != 3, 12]))
    got = n(ops.filter3d(t(pws), t(mixed))).astype(np.float64)
    ok = ~ref["flagged"]
    assert np.all(np.abs(got - ref["filter"])[ok] <= 1e-6 * ref["filter"][ok])


def test_camera_table_from_camera_objects():
    from easygaussiansplatting_b200 import ops
    from easygaussiansplatting_b200.gsfunction import Camera
    table = ring_table(5, seed=4)
    cams = [Camera(r[16], r[17], r[12], r[13], r[14], r[15], t(r[:9].reshape(3, 3)), t(r[9:12])) for r in table]
    assert torch.equal(ops.camera_table(cams), t(table))
    pws = t(box_points(3000, seed=5)[0])
    assert torch.equal(ops.filter3d(pws, cams), ops.filter3d(pws, t(table)))
    cams[2].width = 0
    with pytest.raises(ValueError, match="width and height"):
        ops.camera_table(cams)


@pytest.mark.parametrize("inplace", [False, True])
def test_apply_backward_vs_oracle(inplace):
    from easygaussiansplatting_b200 import ops
    s, a, f, rows = edge_rows(21, n=100003)
    sf, af = ops.filter3d_apply(t(s), t(a), t(f))
    rsf, raf, tt = of3.apply(s, a, f)
    z = rows["zero_f"]
    assert np.array_equal(n(sf)[z], s[z]) and np.array_equal(n(af)[z], a[z])
    assert np.all(np.abs(n(sf) - rsf) <= 4e-7 * rsf)
    assert np.all(np.abs(n(af) - raf) <= 1e-6 * raf + 1e-30)
    rng = np.random.default_rng(22)
    gsf, gaf = rng.normal(size=s.shape).astype(np.float32), rng.normal(size=a.shape).astype(np.float32)
    GS, GA = t(gsf), t(gaf)
    gs, ga = ops.filter3d_backward(t(s), t(a), t(f), GS, GA, inplace=inplace)
    if inplace:
        assert gs.data_ptr() == GS.data_ptr() and ga.data_ptr() == GA.data_ptr()
    rgs, rga = of3.backward(s, a, f, gsf, gaf)
    mag = np.abs(gsf) * tt + np.abs(rgs - gsf * tt) + 1e-30
    assert np.all(np.abs(n(gs) - rgs) <= 2e-6 * mag)
    assert np.all(np.abs(n(ga) - rga) <= 1e-6 * np.abs(rga) + 1e-30)
    assert np.array_equal(n(gs)[z], gsf[z]) and np.array_equal(n(ga)[z], gaf[z])


def _case(N=20000, Wf=640, Hf=360, seed=5):
    sc = synthetic_scene(N, Wf, Hf, sh_dim=12, seed=seed)
    P = {k: t(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    al = t(sc["alphas"][:, None]).requires_grad_()
    us0 = torch.zeros((N, 2), device=DEV, requires_grad=True)
    return sc, P, al, us0


def _cam(sc, Wf, Hf, aa=False, view=None):
    from easygaussiansplatting_b200.gsfunction import Camera
    if view is None:
        R, tc, tw = sc["Rcw"], sc["tcw"], sc["twc"]
    else:
        R, tc, tw = ring_camera(view, 8)
    return Camera(Wf, Hf, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(R), t(tc), t(tw), antialiased=aa)


def _filter(sc, P, Wf, Hf):
    from easygaussiansplatting_b200 import ops
    table = ops.camera_table([_cam(sc, Wf, Hf)] + [_cam(sc, Wf, Hf, view=v) for v in range(4)])
    return ops.filter3d(P["pws"].detach(), table)


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("kind", ["plain", "rgbd", "pose", "rgbd_pose"])
def test_fused_classes_with_filter(kind, aa):
    """Each fused class with a filter: the image is bit-identical to ops.splat on (s', alpha'); the
    gradients equal the same class run unfiltered on leaves s', alpha' (which the existing tests hold to
    the oracle chain) taken through the oracle's filter backward (to the rasterizer backward's
    run-to-run rounding); the filter gets no gradient"""
    from easygaussiansplatting_b200 import gsfunction as G
    from easygaussiansplatting_b200 import ops
    Wf, Hf = 640, 360
    sc, P, al, us0 = _case()
    cam = _cam(sc, Wf, Hf, aa)
    f = _filter(sc, P, Wf, Hf)
    assert (f > 0).all()
    F = {"plain": G.GSFunctionFused, "rgbd": G.GSFunctionFusedRGBD, "pose": G.GSFunctionFusedPose,
         "rgbd_pose": G.GSFunctionFusedRGBDPose}[kind]
    pose = "pose" in kind
    R, tc, tw = (t(sc[k]).requires_grad_() for k in ("Rcw", "tcw", "twc"))
    dl = t(upstream_gradient(Wf, Hf, 3) * (3.0 * Wf * Hf))

    def run(scales, alphas, filt):
        args = (P["pws"], P["shs"], alphas, scales, P["rots"], us0) + ((R, tc, tw) if pose else ()) + (cam,)
        outs = F.apply(*args, *(() if filt is None else (filt,)))
        loss = (outs[0] * dl).sum() + ((outs[1] * 0.01).sum() if "rgbd" in kind else 0.0)
        loss.backward()
        return outs[0].detach()

    f_leaf = f.clone().requires_grad_()
    img = run(P["scales"], al, f_leaf)
    assert f_leaf.grad is None
    got = {k: v.grad.clone() for k, v in P.items()}
    got["alphas"] = al.grad.clone()
    cam_grads = [x.grad.clone() for x in (R, tc, tw)] if pose else []
    sf, af = ops.filter3d_apply(P["scales"].detach(), al.detach(), f)
    pre = ops.preprocess(P["pws"].detach(), P["rots"].detach(), sf, P["shs"].detach(), cam.Rcw, cam.tcw, cam.twc,
                         cam.fx, cam.fy, cam.cx, cam.cy, Wf, Hf, alphas=af, antialiased=aa)
    drawn = pre[6] if aa else af
    ref_img = (ops.splat_rgbd if "rgbd" in kind else ops.splat)(Hf, Wf, *pre[:2], drawn, pre[3], pre[2], pre[4],
                                                                   records=pre[5], capacity=True)[0]
    assert torch.equal(img, ref_img)
    for x in list(P.values()) + [al, us0, R, tc, tw]:
        x.grad = None
    sfl, afl = sf.clone().requires_grad_(), af.clone().requires_grad_()
    img2 = run(sfl, afl, None)
    assert torch.equal(img2, img)
    gs, ga = of3.backward(n(P["scales"]), n(al), n(f), n(sfl.grad), n(afl.grad))
    for k in ("pws", "shs", "rots"):
        assert _rel(got[k], P[k].grad) <= 1e-5, k
    assert _rel(got["scales"], t(gs)) <= 1e-5
    assert _rel(got["alphas"].reshape(-1), t(ga)) <= 1e-5
    for a, b in zip(cam_grads, (R.grad, tc.grad, tw.grad)):
        assert _rel(a, b) <= 1e-4


@pytest.mark.parametrize("kind", ["plain", "rgbd", "pose", "rgbd_pose"])
def test_filter_passed_as_none(kind):
    """filter3d=None passed explicitly (as GraphedFusedStep / MultiViewStep accept it): backward returns
    one gradient per input, and the step is the one without the argument (image bit for bit, gradients
    to the rasterizer backward's run-to-run rounding)"""
    from easygaussiansplatting_b200 import gsfunction as G
    Wf, Hf = 320, 240
    sc, P, al, us0 = _case(N=5000, Wf=Wf, Hf=Hf, seed=12)
    cam = _cam(sc, Wf, Hf)
    F = {"plain": G.GSFunctionFused, "rgbd": G.GSFunctionFusedRGBD, "pose": G.GSFunctionFusedPose,
         "rgbd_pose": G.GSFunctionFusedRGBDPose}[kind]
    R, tc, tw = (t(sc[k]).requires_grad_() for k in ("Rcw", "tcw", "twc"))
    leaves = list(P.values()) + [al] + ([R, tc, tw] if "pose" in kind else [])
    dl = t(upstream_gradient(Wf, Hf, 6) * (3.0 * Wf * Hf))
    res = []
    for extra in ((), (None,)):
        for x in leaves:
            x.grad = None
        args = (P["pws"], P["shs"], al, P["scales"], P["rots"], us0) + ((R, tc, tw) if "pose" in kind else ())
        outs = F.apply(*args, cam, *extra)
        loss = (outs[0] * dl).sum() + ((outs[1] * 0.01).sum() if "rgbd" in kind else 0.0)
        loss.backward()
        res.append([outs[0].detach()] + [x.grad.clone() for x in leaves])
    assert torch.equal(res[0][0], res[1][0])
    for a, b in zip(res[0][1:], res[1][1:]):
        assert _rel(b, a) <= 2e-6


def test_zero_filter_reproduces_todays_step():
    """A zero filter: apply and backward pass their inputs through bit for bit, so the image is
    today's bit for bit, and the gradients are today's up to the rasterizer backward's run-to-run
    rounding (its moment rows are float atomics)"""
    from easygaussiansplatting_b200 import ops
    from easygaussiansplatting_b200.gsfunction import GSFunctionFused
    Wf, Hf = 640, 360
    sc, P, al, us0 = _case(seed=8)
    cam = _cam(sc, Wf, Hf)
    zero = torch.zeros(P["pws"].shape[0], device=DEV)
    sf, af = ops.filter3d_apply(P["scales"].detach(), al.detach(), zero)
    assert torch.equal(bits(sf), bits(P["scales"])) and torch.equal(bits(af), bits(al))
    g = torch.randn_like(sf), torch.randn_like(af)
    gs, ga = ops.filter3d_backward(P["scales"].detach(), al.detach(), zero, *g)
    assert torch.equal(bits(gs), bits(g[0])) and torch.equal(bits(ga), bits(g[1]))
    dl = t(upstream_gradient(Wf, Hf, 2) * (3.0 * Wf * Hf))
    res = []
    for filt in (None, zero):
        for x in list(P.values()) + [al]:
            x.grad = None
        img, _ = GSFunctionFused.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us0, cam,
                                       *(() if filt is None else (filt,)))
        img.backward(dl)
        res.append([img.detach()] + [x.grad.clone() for x in list(P.values()) + [al]])
    assert torch.equal(res[0][0], res[1][0])
    for a, b in zip(res[0][1:], res[1][1:]):
        assert _rel(b, a) <= 2e-6


@pytest.mark.parametrize("aa", [False, True])
def test_graphed_and_multiview_with_filter(aa):
    """GraphedFusedStep with a filter replays the eager filtered step (image bitwise, gradients to the
    rasterizer backward's rounding); MultiViewStep at world 1 sums the eager filtered views"""
    from easygaussiansplatting_b200.graphed import GraphedFusedStep
    from easygaussiansplatting_b200.gsfunction import GSFunctionFused
    from easygaussiansplatting_b200.parallel import MultiViewStep
    Wf, Hf = 320, 240
    sc, P, al, us0 = _case(Wf=Wf, Hf=Hf, seed=6)
    f = _filter(sc, P, Wf, Hf)
    cam = _cam(sc, Wf, Hf, aa)
    dl = t(upstream_gradient(Wf, Hf, 1) * (3.0 * Wf * Hf))
    step = GraphedFusedStep(P["pws"], P["shs"], al, P["scales"], P["rots"], cam, filter3d=f)
    image, _ = GSFunctionFused.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us0, cam, f)
    image.backward(dl)
    assert torch.equal(step.forward(), image.detach())
    step.dloss_dimage.copy_(dl)
    g = step.backward()
    pairs = (("dpws", P["pws"]), ("dshs", P["shs"]), ("dscales", P["scales"]), ("drots", P["rots"]), ("dalphas", al))
    for name, leaf in pairs:
        assert _rel(g[name].reshape(leaf.shape), leaf.grad) <= 2e-6, name
    for x in list(P.values()) + [al]:
        x.grad = None
    cams = [_cam(sc, Wf, Hf, aa, view=v) for v in range(3)]
    dls = [t(upstream_gradient(Wf, Hf, v) * (3.0 * Wf * Hf)) for v in range(3)]
    for c, d in zip(cams, dls):
        im, _ = GSFunctionFused.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us0, c, f)
        im.backward(d)
    mv = MultiViewStep(P["pws"].detach(), P["rots"].detach(), P["scales"].detach(), P["shs"].detach(), al.detach(),
                       filter3d=f)
    lib = _lib.load()
    kid = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())].index("filter3d_apply")
    before = lib.gsb_profile_launches(kid)
    for c, d in zip(cams, dls):
        _, ctx = mv.render(c)
        mv.backward(ctx, d)
    g = mv.reduce()
    assert lib.gsb_profile_launches(kid) - before == 1  # s', alpha' once per step, for all three views
    for name, leaf in pairs:
        assert _rel(g[name].reshape(leaf.shape), leaf.grad) <= 2e-6, name


def test_exchange_with_filter():
    """world 1 through autograd: GSFunctionFused with cam.grad_exchange and a filter returns the
    gradients of the call without the exchange.  World 2 (two ranks on two streams): the filter's
    backward on the exchanged sum equals the sum of each rank's filtered local gradients."""
    from easygaussiansplatting_b200 import ops
    from easygaussiansplatting_b200.gsfunction import GSFunctionFused
    from easygaussiansplatting_b200.parallel import GradExchange
    N, Wf, Hf = 3001, 256, 160
    sc, P, al, us0 = _case(N=N, Wf=Wf, Hf=Hf, seed=4)
    f = _filter(sc, P, Wf, Hf)
    cam = _cam(sc, Wf, Hf)
    dl = t(upstream_gradient(Wf, Hf, 4) * (3.0 * Wf * Hf))
    region, _ = GradExchange.alloc_region(GradExchange.region_bytes(N, 4, 1))
    ex = GradExchange(N, 4, 1, 0, [region], DEV, own_region=region)
    got = {}
    try:
        for mode in ("plain", "exchange"):
            for x in list(P.values()) + [al]:
                x.grad = None
            cam.grad_exchange = ex if mode == "exchange" else None
            img, _ = GSFunctionFused.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us0, cam, f)
            img.backward(dl)
            got[mode] = [x.grad.clone() for x in list(P.values()) + [al]]
        assert ex.status() == 0
        for a, b in zip(got["plain"], got["exchange"]):
            assert _rel(b, a) <= 1e-6
    finally:
        ex.close()
    cam.grad_exchange = None
    world = 2
    pws, rots, shs = (P[k].detach() for k in ("pws", "rots", "shs"))
    sf, af = ops.filter3d_apply(P["scales"].detach(), al.detach(), f)
    regions = [GradExchange.alloc_region(GradExchange.region_bytes(N, 4, world))[0] for _ in range(world)]
    exs = [GradExchange(N, 4, world, r, regions, DEV, own_region=regions[r]) for r in range(world)]
    streams = [torch.cuda.Stream() for _ in range(world)]
    try:
        gen = torch.Generator(device=DEV).manual_seed(7)
        cams, ins, want_s, want_a = [], [], 0, 0
        for r in range(world):
            cams.append(_cam(sc, Wf, Hf, view=r))
            c = cams[r]
            ci = ops.preprocess(pws, rots, sf, shs, c.Rcw, c.tcw, c.twc, c.fx, c.fy, c.cx, c.cy, Wf, Hf)[1]
            m = torch.randn((N, 9), device=DEV, generator=gen)
            ins.append((m, ci))
            out = ops.preprocessB(pws, rots, sf, shs, c.Rcw, c.tcw, c.twc, c.fx, c.fy, c.cx, c.cy, Wf, Hf, None, None,
                                  None, moments=m, cinv2ds=ci)
            gs, ga = ops.filter3d_backward(P["scales"].detach(), al.detach(), f, out[2], out[5])
            want_s, want_a = want_s + gs.double(), want_a + ga.double()
        torch.cuda.synchronize()
        for r in range(world):
            with torch.cuda.stream(streams[r]):
                exs[r].push(pws, rots, sf, shs, cams[r], moments=ins[r][0], cinv2ds=ins[r][1])
        outs = []
        for r in range(world):
            with torch.cuda.stream(streams[r]):
                outs.append(exs[r].reduce())
        torch.cuda.synchronize()
        for r in range(world):
            assert exs[r].status() == 0
            gs, ga = ops.filter3d_backward(P["scales"].detach(), al.detach(), f, outs[r]["dscales"],
                                           outs[r]["dalphas"])
            assert _rel(gs.double(), want_s) <= 1e-6 and _rel(ga.double().reshape(-1), want_a.reshape(-1)) <= 1e-6
    finally:
        for e in exs:
            e.close()


def test_bake_filter3d():
    """The baked parameters' activated scales and opacities are s', alpha' within the exp(log) and
    sigmoid(logit) round trips, and the baked model rendered without the filter matches the filtered
    render.  Tolerance: the round trips move s' and alpha' by a few ulp (relative 2^-21 bounds them),
    which moves a pixel by at most about that relative amount of its value plus the flips of the
    0.002 skip threshold; so the image must agree to 1e-4 on all but 0.1 % of the pixels."""
    from easygaussiansplatting_b200 import gau_io, ops
    from easygaussiansplatting_b200.gsfunction import GSFunctionFused
    Wf, Hf = 640, 360
    sc, P, al, us0 = _case(seed=9)
    N = P["pws"].shape[0]
    params = {"pws": P["pws"].detach(), "low_shs": P["shs"].detach()[:, :3],
              "high_shs": torch.cat([P["shs"].detach()[:, 3:], torch.zeros((N, 36), device=DEV)], 1),
              "alphas_raw": torch.logit(al.detach()), "scales_raw": torch.log(P["scales"].detach()),
              "rots_raw": P["rots"].detach()}
    rows = gau_io.params_to_gs_rows(params)
    s_act, a_act = rows[:, 7:10].contiguous(), rows[:, 10].contiguous()
    f = _filter(sc, P, Wf, Hf)
    sf, af = ops.filter3d_apply(s_act, a_act, f)
    baked = gau_io.bake_filter3d(params, f)
    brows = gau_io.params_to_gs_rows(baked)
    assert _rel(brows[:, 7:10], sf) <= 2 ** -20 and float(((brows[:, 10] - af).abs() / af.clamp_min(1e-30)).max()) \
        <= 2 ** -18
    cam = _cam(sc, Wf, Hf)
    shs = torch.cat([rows[:, 11:14], rows[:, 14:23]], 1)  # SH degree 1 of the scene (12 of 48 columns)
    with torch.no_grad():
        img_f, _ = GSFunctionFused.apply(rows[:, :3], shs, a_act[:, None], s_act, rows[:, 3:7], us0, cam, f)
        img_b, _ = GSFunctionFused.apply(brows[:, :3], torch.cat([brows[:, 11:14], brows[:, 14:23]], 1),
                                         brows[:, 10:11].contiguous(), brows[:, 7:10].contiguous(), brows[:, 3:7],
                                         us0, cam)
    e = (img_f - img_b).abs().amax(0)
    assert float((e > 1e-4).float().mean()) <= 1e-3, float(e.max())
