"""GPU checks of antialiasing (alpha_eff = rho alpha, the 2D-filter opacity compensation):
ops.preprocess(antialiased=True) and every ops.preprocessB form with it against the fp64 oracle
(oracle/aa_oracle.py), bit-level identity of everything antialiasing must not touch, and the
autograd classes, GraphedFusedStep and MultiViewStep with cam.antialiased, plus the refusals."""
import numpy as np
import pytest
import torch

from oracle import aa_oracle as oaa
from oracle import oracle as orc
from oracle import pose_oracle as opose
from easygaussiansplatting_b200.scene import upstream_gradient

from test_antialias_cpu import H, W, edge_scene, oracle_backward, rel_tol
from test_gpu_fused import scene as gpu_scene
from test_gpu_pose import _moment_grads

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).to(DEV)


def n(x):
    return x.detach().cpu().numpy()


def bits(x):
    return x.detach().contiguous().view(torch.int32)


def _params(sc):
    return [t(sc[k]) for k in ("pws", "rots", "scales", "shs", "Rcw", "tcw", "twc")] + \
        [sc["fx"], sc["fy"], sc["cx"], sc["cy"]]


def flagged(sc, s):
    """rows bounded separately (aa_oracle.flagged: the clamp, ill-conditioned 2D or 3D covariances)"""
    return oaa.flagged(sc["scales"], s)


def _grid_scene(N, k3):
    """test_gpu_fused_oracle's scenes (culled and fov-clamped rows, general pose) with the AA edge
    rows of test_antialias_cpu at the head when there is room"""
    if N >= 64:
        sc, _ = edge_scene(k3, seed=N % 1000 + k3, n=N)
    else:
        sc = gpu_scene(N, W, H, 3 * k3, N + k3)
    sc["alphas"] = np.random.default_rng(N + 7 * k3).uniform(0.02, 1.0, N).astype(np.float32)
    return sc


@pytest.mark.parametrize("k3", [1, 4, 9, 16])
@pytest.mark.parametrize("N", [1, 127, 129, 20001])
def test_forward_aa_vs_oracle_and_non_aa_bits(N, k3):
    from easygaussiansplatting_b200 import ops
    sc = _grid_scene(N, k3)
    args = _params(sc) + [W, H]
    al = t(sc["alphas"])
    aa = ops.preprocess(*args, alphas=al, antialiased=True)
    base = ops.preprocess(*args, alphas=al)
    assert len(aa) == 7 and len(base) == 6
    for a, b in zip(aa[:5], base[:5]):  # us, conics, colours, depths, areas
        assert torch.equal(bits(a), bits(b))
    ra, rb = n(aa[5]).view(np.uint32), n(base[5]).view(np.uint32)
    other = [c for c in range(12) if c not in (3, 7)]  # all words but alpha and thr
    assert np.array_equal(ra[:, other], rb[:, other])
    assert np.array_equal(ra[:, 3], n(aa[6]).view(np.uint32))
    st = oaa.stages(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                    sc["fy"], sc["cx"], sc["cy"], W, H)
    s = oaa.scale(st["c2"], st["keep"])
    want = s["rho"] * sc["alphas"]
    got = n(aa[6]).astype(np.float64)
    err = np.abs(got - want)
    flag = flagged(sc, s)
    ok = (err <= want * rel_tol(s)) | flag
    assert ok.all(), (np.flatnonzero(~ok)[:5], err[~ok][:5])
    # flagged rows: still an opacity scaled by a factor in [0.005, 1]
    assert np.all((got[flag] >= 0.0049 * sc["alphas"][flag]) & (got[flag] <= sc["alphas"][flag]))
    if N > 1000:  # binning is the same: tile ranges and sorted ids
        outs = [ops.splat(H, W, x[0], x[1], a, x[3], x[2], x[4], records=x[5])
                for x, a in ((aa, aa[6]), (base, al))]
        assert torch.equal(outs[0][3], outs[1][3]) and torch.equal(outs[0][4], outs[1][4])


def _bwd_case(k3, N=3000):
    sc, rows = edge_scene(k3, seed=90 + k3, n=N)
    rng = np.random.default_rng(k3 + 11)
    sc["alphas"] = rng.uniform(0.05, 1.0, N).astype(np.float32)
    m = rng.normal(size=(N, 9)).astype(np.float32)
    m[::7, :2] = 0
    only = np.arange(16, 64)  # rows whose only upstream gradient is dL/dalpha_eff
    m[only, :5] = 0; m[only, 6:] = 0
    gz = rng.normal(size=N).astype(np.float32)
    gz[only] = 0
    st = oaa.stages(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                    sc["fy"], sc["cx"], sc["cy"], W, H)
    ci = np.ascontiguousarray(st["ci"], dtype=np.float32)
    return sc, rows, m, ci, gz, only


def _ref(sc, m, ci, gz):
    gu, gci, gcol = _moment_grads(m, ci)
    up = (gu.astype(np.float32), gci.astype(np.float32), gcol.astype(np.float32), gz, m[:, 5])
    return oracle_backward(sc, sc["shs"].shape[1] // 3, up)


@pytest.mark.parametrize("k3", [1, 4, 9, 16])
@pytest.mark.parametrize("depth", [False, True])
def test_backward_aa_forms_vs_oracle(k3, depth):
    from easygaussiansplatting_b200 import ops
    sc, rows, m, ci, gz, only = _bwd_case(k3)
    N = len(sc["pws"])
    args = _params(sc) + [W, H, None, None, None]
    kw = dict(moments=t(m), cinv2ds=t(ci), dloss_ddepths=t(gz) if depth else None)
    al = t(sc["alphas"])
    out = ops.preprocessB(*args, **kw, antialiased=True, alphas=al)
    ref, st, s, gc2 = _ref(sc, m, ci, gz if depth else np.zeros(N, np.float32))
    flag = flagged(sc, s)
    got = dict(pws=out[0], shs=out[1], scales=out[2], rots=out[3])
    for name, g in got.items():
        g = n(g).astype(np.float64).reshape(ref[name].shape)
        e = np.abs(g - ref[name])[~flag].max() / np.abs(ref[name]).max()
        assert e < 3e-5, (name, e)
        assert np.isfinite(g).all()
    dal = n(out[5]).astype(np.float64)
    assert np.all((np.abs(dal - ref["alphas"]) <= rel_tol(s) * np.abs(ref["alphas"])) | s["near"])
    # dL/dalpha_eff alone moves the geometry of kept, unclamped rows
    live = only[st["keep"][only] & ~s["clamped"][only]]
    assert len(live) > 10 and (n(out[2])[live] != 0).any(1).all()
    # clamped rows (zero scale): 0.005 m[5] for alpha and the non-AA geometry gradient
    z = rows["zero"]
    base = ops.preprocessB(*args, **kw)
    assert np.array_equal(n(out[5])[z], (np.float32(np.sqrt(np.float32(2.5e-5))) * m[z, 5]).astype(np.float32))
    for a, b in zip(out[:4], base[:4]):
        assert np.allclose(n(a)[z], n(b)[z], rtol=1e-6, atol=1e-6 * float(n(b).__abs__().max()))
    assert torch.equal(bits(out[4]), bits(base[4]))  # dL/du is not touched
    # antialiased=False is today's call, bit for bit
    off = ops.preprocessB(*args, **kw, antialiased=False, alphas=al)
    for a, b in zip(off, base):
        assert torch.equal(bits(a), bits(b))
    # compact: the same small gradients, no dL/dsh row
    cp = ops.preprocessB(*args, **kw, compact=True, antialiased=True, alphas=al)
    assert cp[1] is None
    for i in (0, 2, 3, 4, 5):
        assert torch.equal(bits(cp[i]), bits(out[i]))
    # camera gradient: the oracle's plus the AA addend; per-Gaussian outputs unchanged; pose only
    pz = ops.preprocessB(*args, **kw, camera_grad=True, antialiased=True, alphas=al)
    g = np.concatenate([n(x).reshape(-1) for x in pz[-1]]).astype(np.float64)
    want = ref["cam"][~flag].sum(0) + ref["cam"][flag].sum(0)
    absum = np.abs(ref["cam"]).sum(0)
    assert (np.abs(g - want) <= 1e-5 * absum + 1e-3 * np.abs(ref["cam"][flag]).sum(0)).all()
    for a, b in zip(pz[:-1], out):
        assert torch.equal(bits(a), bits(b))
    po = ops.preprocessB(*args, **kw, camera_grad=True, pose_only=True, antialiased=True, alphas=al)
    assert all(x is None for x in po[:-1])
    for a, b in zip(po[-1], pz[-1]):
        assert torch.equal(bits(a), bits(b))


def _autograd_case(N, Wf, Hf, sh_dim, seed):
    sc = gpu_scene(N, Wf, Hf, sh_dim, seed)
    P = {k: t(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    al = t(sc["alphas"][:, None]).requires_grad_()
    us0 = torch.zeros((N, 2), device=DEV, requires_grad=True)
    return sc, P, al, us0


@pytest.mark.parametrize("rgbd", [False, True])
@pytest.mark.parametrize("N,Wf,Hf", [(20000, 979, 546), (100000, 1600, 900)])
def test_fused_classes_antialiased_vs_oracle(rgbd, N, Wf, Hf):
    """GSFunctionFused / GSFunctionFusedRGBD with cam.antialiased: the image is the oracle renderer's
    fed the oracle's alpha_eff, and the colour gradients are the oracle's splat_backward (on alpha_eff)
    through the chain plus the AA term"""
    from easygaussiansplatting_b200 import ops
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused, GSFunctionFusedRGBD
    sc, P, al, us0 = _autograd_case(N, Wf, Hf, 12, 5)
    cam = Camera(Wf, Hf, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]),
                 antialiased=True)
    F = GSFunctionFusedRGBD if rgbd else GSFunctionFused
    outs = F.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us0, cam)
    dl = t(upstream_gradient(Wf, Hf, 3) * (3.0 * Wf * Hf))
    outs[0].backward(dl)
    # the same frame through the ops: the image is bit-identical
    pre = ops.preprocess(*_params(sc), Wf, Hf, alphas=al.detach(), antialiased=True)
    img = (ops.splat_rgbd if rgbd else ops.splat)(Hf, Wf, *pre[:2], pre[6], pre[3], pre[2], pre[4],
                                                   records=pre[5], capacity=True)[0]
    assert torch.equal(img, outs[0].detach())
    # the oracle
    st = oaa.stages(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                    sc["fy"], sc["cx"], sc["cy"], Wf, Hf)
    s = oaa.scale(st["c2"], st["keep"])
    flag = flagged(sc, s)
    # the rasterizers are checked on the kernel's alpha_eff (test_forward_aa_vs_oracle_and_non_aa_bits
    # holds it to the oracle's): a relative 1e-3 of rho on an ill-conditioned row would otherwise
    # move pixels across the 0.002 threshold the oracle flags on its own values
    alpha_eff = n(pre[6])
    assert np.all((np.abs(alpha_eff - s["rho"] * sc["alphas"]) <= s["rho"] * sc["alphas"] * rel_tol(s)) | flag)
    # ... and on the kernel's per-Gaussian outputs (the stages are held to the oracle's elsewhere)
    us_k, ci_k, col_k = n(pre[0]), n(pre[1]), n(pre[2])
    fwd = orc.splat(Hf, Wf, us_k, ci_k, alpha_eff, n(pre[3]).copy(), col_k, n(pre[4]).copy())
    amb = fwd["ambiguous"]
    e = np.abs(n(outs[0]) - fwd["image"]).max(0)
    assert e[~amb].max() < 2e-4 and (amb.mean() < 0.01)
    if not rgbd:
        du, dc, da, dcol = orc.splat_backward(Hf, Wf, us_k, ci_k, alpha_eff, col_k, fwd, n(dl))
        ref = orc.chain_backward(sc["Rcw"], du, dc, da, dcol, *st["J"])
        gc2 = oaa.dcov2d_addend(st["c2"], st["keep"], sc["alphas"], da.reshape(-1))
        add = oaa.chain(st, sc["Rcw"], gc2)
        for name, g in (("pws", P["pws"].grad), ("scales", P["scales"].grad), ("rots", P["rots"].grad)):
            want = ref[name] + add[name]
            err = np.abs(n(g).astype(np.float64) - want)[~flag]
            assert np.quantile(err / np.abs(want).max(), 0.999) < 1e-3, name
        want = s["rho"] * da.reshape(-1)
        got = n(al.grad).reshape(-1)
        assert np.quantile(np.abs(got - want) / np.abs(want).max(), 0.999) < 1e-3


def test_pose_class_antialiased_vs_oracle():
    """GSFunctionFusedPose with cam.antialiased: its camera gradient is the pose oracle's of the same
    rasterizer gradients plus the AA addend's"""
    from easygaussiansplatting_b200 import ops
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFusedPose
    Wf, Hf = 640, 360
    sc, P, al, us0 = _autograd_case(20000, Wf, Hf, 12, 7)
    R, tc, tw = (t(sc[k]).requires_grad_() for k in ("Rcw", "tcw", "twc"))
    cam = Camera(Wf, Hf, sc["fx"], sc["fy"], sc["cx"], sc["cy"], R.detach(), tc.detach(), tw.detach(),
                 antialiased=True)
    image, _ = GSFunctionFusedPose.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us0, R, tc, tw, cam)
    dl = t(upstream_gradient(Wf, Hf, 4) * (3.0 * Wf * Hf))
    image.backward(dl)
    # the same rasterizer gradients through ops.preprocessB(camera_grad=True, antialiased=True)
    pre = ops.preprocess(*_params(sc), Wf, Hf, alphas=al.detach(), antialiased=True)
    f = ops.splat(Hf, Wf, *pre[:2], pre[6], pre[3], pre[2], pre[4], records=pre[5], capacity=True)
    mom = ops.splatB(Hf, Wf, pre[0], pre[1], pre[6], pre[3], pre[2], *f[1:5], dl, moments_only=True)
    m = n(mom)
    st = oaa.stages(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                    sc["fy"], sc["cx"], sc["cy"], Wf, Hf)
    gu, gci, gcol = _moment_grads(m, n(pre[1]))
    per = opose.camera_grad(st, sc["pws"], sc["Rcw"], sc["fx"], sc["fy"], Wf, Hf, gu, gci, gcol)["per"]
    per = per + oaa.camera(st, sc["pws"], sc["Rcw"], sc["fx"], sc["fy"], Wf, Hf,
                           oaa.dcov2d_addend(st["c2"], st["keep"], sc["alphas"], m[:, 5]))
    g = np.concatenate([n(R.grad).reshape(-1), n(tc.grad), n(tw.grad)]).astype(np.float64)
    absum = np.abs(per).sum(0)
    assert (np.abs(g - per.sum(0)) <= 1e-4 * absum).all(), np.abs(g - per.sum(0)) / absum


def test_graphed_and_multiview_antialiased():
    """GraphedFusedStep with cam.antialiased replays the eager AA step (image bitwise, gradients to the
    rasterizer backward's run-to-run rounding); MultiViewStep at world 1 sums the single-view AA
    gradients"""
    from easygaussiansplatting_b200.graphed import GraphedFusedStep
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused
    from easygaussiansplatting_b200.parallel import MultiViewStep
    from easygaussiansplatting_b200.scene import ring_camera
    N, Wf, Hf = 20000, 320, 240
    sc, P, al, us0 = _autograd_case(N, Wf, Hf, 12, 6)
    cam = Camera(Wf, Hf, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]),
                 antialiased=True)
    dl = t(upstream_gradient(Wf, Hf, 1) * (3.0 * Wf * Hf))
    step = GraphedFusedStep(P["pws"], P["shs"], al, P["scales"], P["rots"], cam)
    image, _ = GSFunctionFused.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us0, cam)
    image.backward(dl)
    img = step.forward()
    assert torch.equal(img, image.detach())
    step.dloss_dimage.copy_(dl)
    g = step.backward()
    for name, ref in (("dpws", P["pws"].grad), ("dshs", P["shs"].grad), ("dscales", P["scales"].grad),
                      ("drots", P["rots"].grad), ("dalphas", al.grad.reshape(-1))):
        err = float((g[name].reshape(ref.shape) - ref).abs().max() / ref.abs().max().clamp_min(1e-30))
        assert err <= 2e-6, (name, err)
    # multi-view
    for p in list(P.values()) + [al]:
        p.grad = None
    cams, dls = [], []
    for v in range(3):
        Rcw, tcw, twc = ring_camera(v, 8)
        cams.append(Camera(Wf, Hf, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(Rcw), t(tcw), t(twc), antialiased=True))
        dls.append(t(upstream_gradient(Wf, Hf, v) * (3.0 * Wf * Hf)))
    for c, d in zip(cams, dls):
        im, _ = GSFunctionFused.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us0, c)
        im.backward(d)
    mv = MultiViewStep(P["pws"].detach(), P["rots"].detach(), P["scales"].detach(), P["shs"].detach(), al.detach())
    for c, d in zip(cams, dls):
        _, ctx = mv.render(c)
        mv.backward(ctx, d)
    g = mv.reduce()
    for name, want in (("dpws", P["pws"].grad), ("dshs", P["shs"].grad), ("dscales", P["scales"].grad),
                       ("drots", P["rots"].grad), ("dalphas", al.grad.reshape(-1))):
        err = float((g[name].reshape(want.shape) - want).abs().max() / want.abs().max().clamp_min(1e-30))
        assert err <= 2e-6, (name, err)


def test_refusals():
    """the seven-operator surface and the gradient exchange have no antialiased form: ValueError"""
    from easygaussiansplatting_b200 import gsfunction
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused
    from easygaussiansplatting_b200.parallel import GradExchange
    sc, P, al, us0 = _autograd_case(500, 64, 64, 3, 2)
    cam = Camera(64, 64, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]),
                 antialiased=True)
    with pytest.raises(ValueError, match="antialiased"):
        gsfunction.GSFunction.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us0, cam)
    with pytest.raises(ValueError, match="antialiased"):
        GradExchange.push(object(), P["pws"], P["rots"], P["scales"], P["shs"], cam)
    cam.grad_exchange = object()
    with pytest.raises(ValueError, match="antialiased"):
        GSFunctionFused.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us0, cam)
