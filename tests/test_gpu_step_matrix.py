"""Every fused training step against one fp64 whole-step oracle (oracle/step_oracle.py): the four
autograd classes x antialiasing x the 3D filter x every SH degree, on a scene with culled, fov-clamped,
zero-scale, needle and huge rows, filter edge rows and a general camera; which backward runs under
needs_input_grad; and GraphedFusedStep / MultiViewStep held to the oracle directly.

The oracle renders on the kernel's own fp32 per-Gaussian outputs (us, conics, colours, depths, the
composited opacities), so that the rasterizer's threshold decisions are taken on the values the device
drew; ops.preprocess is held to the oracle's stages elsewhere.  Its Jacobians are its own.  Bounds, per
parameter, with the error of a row its largest entry error over max|ref|: 1e-4 on rows step_oracle does
not flag, 5e-3 on every row outside the near-plane band that is not thin (aa_oracle.thin); the camera
gradient to 1e-4 absum plus 5e-3 of the flagged rows' sum |per| (the oracle's rasterizer backward is in
the loop) plus the thin rows' own sum |per|."""
import numpy as np
import pytest
import torch

from oracle import filter3d_oracle as of3
from oracle import step_oracle as ost
from easygaussiansplatting_b200.scene import ring_camera, upstream_gradient

from test_antialias_cpu import aa_edge_rows
from test_filter3d_cpu import camera_row, ring_table
from test_gpu_fused import scene as gpu_scene
from test_gpu_pose import _Moments

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KINDS = ("plain", "rgbd", "pose", "rgbd_pose")
K3S = (1, 4, 9, 16)
N_MAT = 20001
GRADS = ("pws", "shs", "scales", "rots", "alphas", "us")


def t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).to(DEV)


def n(x):
    return x.detach().cpu().numpy()


def bits(x):
    return x.detach().contiguous().view(torch.int32)


def matrix_scene(N, W, H, k3, seed):
    """test_gpu_fused.scene (culled and fov-clamped rows; an odd seed: a general pose) with
    test_antialias_cpu's AA edge rows at 0-15 (zero scale, needles, huge, culled) and filter edge rows:
    16-19 f = 0, 20-23 f = 1e3 s_max and 32-35 one zero scale axis under f > 0 (alpha' ~ 0 and = 0:
    never composited, so no gradient at all), 24-27 isotropic with f = 3 s (s' ~ f, drawn), 28-31
    f = 1e-3 s_min.
    The filter is the oracle's of a ring of cameras plus the render camera, rounded to fp32 (ops.filter3d
    is held to it elsewhere).  -> (scene, filter[N] f32, rows)"""
    sc = gpu_scene(N, W, H, 3 * k3, seed)
    sc, rows = aa_edge_rows(sc)
    rng = np.random.default_rng(seed + 11)
    sc["alphas"] = rng.uniform(0.05, 1.0, N).astype(np.float32)
    table = np.concatenate([ring_table(8, seed=seed),
                            camera_row(sc["Rcw"], sc["tcw"], sc["fx"], sc["fy"], sc["cx"], sc["cy"], W, H)[None]])
    f = of3.filter3d(sc["pws"], table)["filter"].astype(np.float32)
    s = sc["scales"]
    f[16:20] = 0.0
    f[20:24] = 1e3 * s[20:24].max(1)
    s[24:28] = s[24:28].max(1, keepdims=True)  # isotropic, so that alpha' = alpha / 10^1.5 is still drawn
    sc["alphas"][24:28] = 0.95
    f[24:28] = 3.0 * s[24:28, 0]
    f[28:32] = 1e-3 * s[28:32].min(1)
    s[32:36, 0] = 0.0
    rows.update(f_zero=np.arange(16, 20), f_huge=np.arange(20, 24), f_big=np.arange(24, 28),
                f_small=np.arange(28, 32), zero_axis=np.arange(32, 36))
    assert (f[32:36] > 0).all()
    return sc, f, rows


def _camera(sc, W, H, aa, pose_of=None):
    from easygaussiansplatting_b200.gsfunction import Camera
    R, tc, tw = pose_of if pose_of is not None else (sc["Rcw"], sc["tcw"], sc["twc"])
    return Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(R), t(tc), t(tw), antialiased=aa)


def _upstream(W, H, seed):
    rng = np.random.default_rng(seed + 77)
    dl = upstream_gradient(W, H, seed) * np.float32(3.0 * W * H)
    return dl, (rng.normal(size=(H, W)) * 0.3).astype(np.float32), rng.normal(size=(H, W)).astype(np.float32)


def run_class(kind, sc, cam, f, flat, dl, dld, dla, need_map=True, need_pose=True):
    """one step of the class through autograd -> (outputs, gradient dict, alpha leaf)"""
    from easygaussiansplatting_b200 import gsfunction as G
    F = {"plain": G.GSFunctionFused, "rgbd": G.GSFunctionFusedRGBD, "pose": G.GSFunctionFusedPose,
         "rgbd_pose": G.GSFunctionFusedRGBDPose}[kind]
    pose, rgbd = "pose" in kind, "rgbd" in kind
    P = {k: t(sc[k]).requires_grad_(need_map) for k in ("pws", "shs", "scales", "rots")}
    al = t(sc["alphas"] if flat else sc["alphas"][:, None]).requires_grad_(need_map)
    us0 = torch.zeros((len(sc["pws"]), 2), device=DEV, requires_grad=need_map)
    R, tc, tw = (t(sc[k]).requires_grad_(pose and need_pose) for k in ("Rcw", "tcw", "twc"))
    args = (P["pws"], P["shs"], al, P["scales"], P["rots"], us0) + ((R, tc, tw) if pose else ()) + (cam,)
    outs = F.apply(*args, *(() if f is None else (t(f),)))
    loss = (outs[0] * t(dl)).sum()
    if rgbd:
        loss = loss + (outs[1] * t(dld)).sum() + (outs[2] * t(dla)).sum()
    loss.backward()
    g = dict(pws=P["pws"].grad, shs=P["shs"].grad, scales=P["scales"].grad, rots=P["rots"].grad, alphas=al.grad,
             us=us0.grad)
    if pose:
        g.update(Rcw=R.grad, tcw=tc.grad, twc=tw.grad)
    return outs, g, al


def drawn_frame(sc, cam, f, rgbd):
    """the frame through the ops (ops.preprocess on ops.filter3d_apply's s', alpha') -> (the kernel's fp32
    per-Gaussian inputs of the rasterizer, the ops' frame)"""
    from easygaussiansplatting_b200 import ops
    s, a = t(sc["scales"]), t(sc["alphas"])
    if f is not None:
        s, a = ops.filter3d_apply(s, a, t(f))
    pre = ops.preprocess(t(sc["pws"]), t(sc["rots"]), s, t(sc["shs"]), cam.Rcw, cam.tcw, cam.twc, cam.fx, cam.fy,
                         cam.cx, cam.cy, cam.width, cam.height, alphas=a, antialiased=cam.antialiased)
    drawn = pre[6] if cam.antialiased else a
    inp = dict(us=n(pre[0]), ci=n(pre[1]), col=n(pre[2]), depths=n(pre[3]), areas=n(pre[4]), alphas=n(drawn))
    splat = ops.splat_rgbd if rgbd else ops.splat
    out = splat(cam.height, cam.width, pre[0], pre[1], drawn, pre[3], pre[2], pre[4], records=pre[5], capacity=True)
    return inp, out


def check_planes(got, o, rgbd):
    amb = o["ambiguous"]
    assert amb.mean() < 0.01, amb.mean()
    # the thin rows (aa_oracle.thin: the needles) and their footprints are bounded separately; they may
    # cover at most 0.1 % of the rows and 2 % of the frame
    assert o["thin"].sum() <= 1e-3 * len(o["thin"]) and o["thin_pixels"].mean() <= 0.02
    amb = amb | o["thin_pixels"]
    planes = [("image", got[0], o["image"])]
    if rgbd:
        planes += [("depth", got[1], o["depth"]), ("alpha", got[2], o["alpha"])]
    for name, g, want in planes:
        e = np.abs(n(g).astype(np.float64) - want)
        e = e.max(0) if e.ndim == 3 else e
        bad = np.argmax(np.where(amb, 0.0, e))
        assert e[~amb].max() <= 2e-4, (name, e[~amb].max(), np.unravel_index(bad, e.shape))


def check_grads(got, want, flagged, band, thin, names=GRADS):
    """thin rows (aa_oracle.thin, at most 0.1 % of them): fp32 keeps ~2^-24 s_max^2 / s_min^2 of their
    thin axes, a relative 0.24 on the needles, so no bound below that means anything; they must be finite"""
    N = len(flagged)
    assert thin.sum() <= 1e-3 * N
    for k in names:
        g = np.asarray(got[k], np.float64).reshape(N, -1)
        w = np.asarray(want[k], np.float64).reshape(N, -1)
        assert np.isfinite(g).all(), k
        err = np.abs(g - w).max(1) / max(np.abs(w).max(), 1e-30)
        assert err[~flagged].max(initial=0) <= 1e-4, (k, err[~flagged].max(initial=0), np.argmax(err * ~flagged))
        loose = ~(band | thin)
        assert err[loose].max(initial=0) <= 5e-3, (k, err[loose].max(initial=0), np.argmax(err * loose))


def check_camera(g15, o):
    """1e-4 absum + 5e-3 of the flagged rows' sum |per|, plus the thin rows' sum |per| itself: fp32 does
    not resolve their thin axes (check_grads), so their camera rows are bounded by their own size
    (measured: 8 % of it on the needles)"""
    per, fl, thin = o["per"], o["flagged"], o["thin"]
    tol = 1e-4 * o["absum"] + 5e-3 * np.abs(per[fl & ~thin]).sum(0) + np.abs(per[thin]).sum(0)
    err = np.abs(np.asarray(g15, np.float64) - o["cam_grad"])
    assert (err <= tol).all(), err / np.maximum(o["absum"], 1e-30)


# ---------------------------------------------------------------- the matrix
CASES = [(kind, aa, filt, k3, 640, 360) for kind in KINDS for aa in (False, True) for filt in (False, True)
         for k3 in K3S] + [(kind, aa, filt, 4, 979, 546) for kind in KINDS for aa in (False, True)
                           for filt in (False, True)]


@pytest.mark.parametrize("kind,aa,filt,k3,W,H", CASES)
def test_class_step_vs_oracle(kind, aa, filt, k3, W, H):
    i = CASES.index((kind, aa, filt, k3, W, H))
    flat = i % 2 == 1  # alphas as [N] in half the cases, [N, 1] in the other half
    sc, f, rows = matrix_scene(N_MAT, W, H, k3, seed=2 * i + 1)
    f = f if filt else None
    pose, rgbd = "pose" in kind, "rgbd" in kind
    dl, dld, dla = _upstream(W, H, i)
    cam = _camera(sc, W, H, aa)
    outs, g, al = run_class(kind, sc, cam, f, flat, dl, dld, dla)
    assert g["alphas"].shape == al.shape
    inp, ref = drawn_frame(sc, cam, f, rgbd)
    assert torch.equal(bits(outs[0]), bits(ref[0]))
    if rgbd:
        assert torch.equal(bits(outs[1]), bits(ref[5])) and torch.equal(bits(outs[2]), bits(ref[6]))
    o = ost.step(sc, ost.camera(sc, W, H), rgbd=rgbd, pose=pose, aa=aa, filt=f, dl=dl,
                 dld=dld if rgbd else None, dla=dla if rgbd else None, drawn_inputs=inp)
    check_planes(outs, o, rgbd)
    got = {k: n(g[k]) for k in GRADS}
    check_grads(got, o["grads"], o["flagged"], o["band"], o["thin"])
    if pose:
        check_camera(np.concatenate([n(g["Rcw"]).reshape(-1), n(g["tcw"]), n(g["twc"])]), o)
    if filt:  # rows never composited (alpha' ~ 0 or = 0): no gradient at all, here or in the oracle
        dead = np.concatenate([rows["f_huge"], rows["zero_axis"]])
        for k in GRADS:
            assert not got[k].reshape(N_MAT, -1)[dead].any(), k
            assert not o["grads"][k].reshape(N_MAT, -1)[dead].any(), k
        assert (np.abs(got["scales"][rows["f_big"]]).sum(1) > 0).any()


# ---------------------------------------------------------------- which backward runs
@pytest.mark.parametrize("filt", [False, True])
@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("kind", ["pose", "rgbd_pose"])
def test_needs_input_grad(monkeypatch, kind, aa, filt):
    """With the same moment rows (test_gpu_pose._Moments): a frozen map runs the pose-only kernel and
    gets the full backward's camera gradient bit for bit; a pose that needs no gradient gets the
    gradients of the class without a pose, bit for bit"""
    W, H, k3 = 640, 360, 4
    sc, f, _ = matrix_scene(N_MAT, W, H, k3, seed=101)
    f = f if filt else None
    dl, dld, dla = _upstream(W, H, 5)
    cam = _camera(sc, W, H, aa)
    rec = _Moments(monkeypatch)
    _, full, _ = run_class(kind, sc, cam, f, False, dl, dld, dla)
    assert rec.saved is not None
    _, po, _ = run_class(kind, sc, cam, f, False, dl, dld, dla, need_map=False)
    for k in GRADS:
        assert po[k] is None, k
    for k in ("Rcw", "tcw", "twc"):
        assert torch.equal(bits(po[k]), bits(full[k])), k
    _, nopose, _ = run_class(kind, sc, cam, f, False, dl, dld, dla, need_pose=False)
    _, plain, _ = run_class(kind.replace("pose", "").rstrip("_") or "plain", sc, cam, f, False, dl, dld, dla)
    for k in GRADS:
        assert torch.equal(bits(nopose[k]), bits(full[k])), k
        assert torch.equal(bits(plain[k]), bits(full[k])), k
    assert all(nopose[k] is None for k in ("Rcw", "tcw", "twc"))


# ---------------------------------------------------------------- the captured and the multi-view step
@pytest.mark.parametrize("filt", [False, True])
@pytest.mark.parametrize("aa", [False, True])
def test_graphed_step_vs_oracle(aa, filt):
    from easygaussiansplatting_b200.graphed import GraphedFusedStep
    W, H, k3 = 640, 360, 16
    sc, f, _ = matrix_scene(N_MAT, W, H, k3, seed=201 + 2 * aa + 4 * filt)
    f = f if filt else None
    dl, _, _ = _upstream(W, H, 7)
    cam = _camera(sc, W, H, aa)
    al = t(sc["alphas"] if filt else sc["alphas"][:, None])
    step = GraphedFusedStep(t(sc["pws"]), t(sc["shs"]), al, t(sc["scales"]), t(sc["rots"]), cam,
                            filter3d=None if f is None else t(f))
    img = step.forward()
    inp, ref = drawn_frame(sc, cam, f, False)
    assert torch.equal(bits(img), bits(ref[0]))
    step.dloss_dimage.copy_(t(dl))
    g = step.backward()
    got = {k: n(g["d" + k]) for k in GRADS}
    o = ost.step(sc, ost.camera(sc, W, H), rgbd=False, pose=False, aa=aa, filt=f, dl=dl, drawn_inputs=inp)
    check_planes([img], o, False)
    check_grads(got, o["grads"], o["flagged"], o["band"], o["thin"])


@pytest.mark.parametrize("filt", [False, True])
@pytest.mark.parametrize("aa", [False, True])
def test_multiview_step_vs_oracle(aa, filt):
    """three views at world 1: the oracle's gradients summed over the views (dL/dsh from
    sh_grad_expand), and each view's own dL/du"""
    from easygaussiansplatting_b200.parallel import MultiViewStep
    W, H, k3 = 640, 360, 16
    sc, f, _ = matrix_scene(N_MAT, W, H, k3, seed=301 + 2 * aa + 4 * filt)
    f = f if filt else None
    al = t(sc["alphas"] if aa else sc["alphas"][:, None])
    mv = MultiViewStep(t(sc["pws"]), t(sc["rots"]), t(sc["scales"]), t(sc["shs"]), al,
                       filter3d=None if f is None else t(f))
    views = []
    for v in range(3):
        R, tc, tw = ring_camera(v, 8)
        vsc = dict(sc, Rcw=R, tcw=tc, twc=tw)
        cam = _camera(vsc, W, H, aa)
        dl, _, _ = _upstream(W, H, 10 + v)
        image, ctx = mv.render(cam)
        inp, ref = drawn_frame(vsc, cam, f, False)
        assert torch.equal(bits(image), bits(ref[0]))
        mv.backward(ctx, t(dl))
        o = ost.step(vsc, ost.camera(vsc, W, H), rgbd=False, pose=False, aa=aa, filt=f, dl=dl, drawn_inputs=inp)
        check_planes([image], o, False)
        views.append(o)
    g = mv.reduce()
    want = {k: sum(o["grads"][k] for o in views) for k in GRADS if k != "us"}
    flagged = np.any([o["flagged"] for o in views], axis=0)
    band = np.any([o["band"] for o in views], axis=0)
    thin = np.any([o["thin"] for o in views], axis=0)
    check_grads({k: n(g["d" + k]) for k in want}, want, flagged, band, thin, names=tuple(want))
    for v, o in enumerate(views):
        check_grads({"us": n(g["dus"][v])}, o["grads"], o["flagged"], o["band"], o["thin"], names=("us",))
