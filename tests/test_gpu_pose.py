"""GPU checks of the camera gradient: ops.preprocessB(camera_grad=True) and the pose-only kernel
against the fp64 pose oracle, bit-level properties (per-Gaussian outputs unchanged, pose-only
writes nothing, run-to-run identical), argument errors, the autograd classes
GSFunctionFusedPose / GSFunctionFusedRGBDPose, and a short RGB-D tracking run."""
import ctypes as C
import functools
import math

import numpy as np
import pytest
import torch

from oracle import pose_oracle as opose
from easygaussiansplatting_b200.scene import synthetic_scene, upstream_gradient

from test_gpu_fused import scene as gpu_scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).to(DEV)


def n(x):
    return x.detach().cpu().numpy()


def bits(x):
    return x.detach().contiguous().view(torch.int32)


@functools.lru_cache(maxsize=2)
def _case(N, k3):
    """a culled, fov-clamped scene with a general pose (odd seed), its oracle stages and random
    upstream gradients (plain and as moment rows)"""
    W, H = 640, 360
    sc = gpu_scene(N, W, H, 3 * k3, 2 * (N % 1000) + 2 * k3 + 1)
    st = opose.stages(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                      sc["fy"], sc["cx"], sc["cy"], W, H)
    rng = np.random.default_rng(N + k3)
    up = dict(gu=rng.normal(size=(N, 2)).astype(np.float32), gci=rng.normal(size=(N, 3)).astype(np.float32),
              gcol=rng.normal(size=(N, 3)).astype(np.float32), gz=rng.normal(size=N).astype(np.float32))
    m = rng.normal(size=(N, 9)).astype(np.float32)
    m[::7, :2] = 0  # untouched rows: dL/du = 0
    up["moments"] = m
    up["cinv2ds"] = np.ascontiguousarray(st["ci"], dtype=np.float32)
    return sc, st, up, W, H


def _moment_grads(m, ci):
    """dL/du, dL/dconic, dL/dcolour from moment rows, as the MOM kernels convert them"""
    m, ci = m.astype(np.float64), ci.astype(np.float64)
    none = (m[:, 0] == 0) & (m[:, 1] == 0)
    gu = -np.stack([ci[:, 0] * m[:, 0] + ci[:, 1] * m[:, 1], ci[:, 1] * m[:, 0] + ci[:, 2] * m[:, 1]], 1)
    gu[none] = 0
    gci = np.stack([-0.5 * m[:, 2], -m[:, 3], -0.5 * m[:, 4]], 1)
    return gu, gci, m[:, 6:9]


def _run(sc, W, H, up, mom, depth, **kw):
    from easygaussiansplatting_b200 import ops
    args = [t(sc[k]) for k in ("pws", "rots", "scales", "shs", "Rcw", "tcw", "twc")]
    args += [sc["fx"], sc["fy"], sc["cx"], sc["cy"], W, H]
    gz = t(up["gz"]) if depth else None
    if mom:
        return ops.preprocessB(*args, None, None, None, moments=t(up["moments"]), cinv2ds=t(up["cinv2ds"]),
                               dloss_ddepths=gz, **kw)
    return ops.preprocessB(*args, t(up["gu"]), t(up["gci"]), t(up["gcol"]), dloss_ddepths=gz, **kw)


def _ref(sc, st, up, W, H, mom, depth):
    if mom:
        gu, gci, gcol = _moment_grads(up["moments"], up["cinv2ds"])
    else:
        gu, gci, gcol = up["gu"], up["gci"], up["gcol"]
    return opose.camera_grad(st, sc["pws"], sc["Rcw"], sc["fx"], sc["fy"], W, H, gu, gci, gcol,
                             up["gz"] if depth else None)


@pytest.mark.parametrize("depth", [False, True])
@pytest.mark.parametrize("mom", [False, True])
@pytest.mark.parametrize("k3", [1, 4, 9, 16])
@pytest.mark.parametrize("N", [1, 127, 128, 129, 20001, 1000000])
def test_camera_grad_vs_oracle(N, k3, mom, depth):
    sc, st, up, W, H = _case(N, k3)
    out = _run(sc, W, H, up, mom, depth, camera_grad=True)
    dR, dt, dw = out[-1]
    g = np.concatenate([n(dR).reshape(-1), n(dt), n(dw)]).astype(np.float64)
    ref = _ref(sc, st, up, W, H, mom, depth)
    err = np.abs(g - ref["grad"])
    assert (err <= 1e-5 * ref["absum"]).all(), (err / np.maximum(ref["absum"], 1e-30)).max()
    if st["keep"].any():
        assert np.abs(g[:12]).max() > 0
    assert dR.shape == (3, 3) and dt.shape == (3,) and dw.shape == (3,)
    # the per-Gaussian outputs are those of the call without camera_grad, bit for bit
    base = _run(sc, W, H, up, mom, depth)
    assert len(out) == len(base) + 1
    for a, b in zip(out[:-1], base):
        assert torch.equal(bits(a), bits(b))
    # pose only: the same camera gradient, no per-Gaussian outputs
    po = _run(sc, W, H, up, mom, depth, camera_grad=True, pose_only=True)
    assert all(x is None for x in po[:-1])
    for a, b in zip(po[-1], out[-1]):
        assert torch.equal(bits(a), bits(b))


def _abi_args(sc, W, H, up, mom, depth, keep):
    """gsb_preprocess_backward_pose's arguments up to dloss_ddepths; `keep` holds the tensors"""
    k3 = sc["shs"].shape[1] // 3
    T = {k: t(sc[k]) for k in ("pws", "rots", "scales", "shs", "Rcw", "tcw", "twc")}
    for k in ("gu", "gci", "gcol", "gz", "moments", "cinv2ds"):
        T[k] = t(up[k])
    keep.update(T)
    p = lambda k: T[k].data_ptr()
    args = [len(sc["pws"]), k3] + [p(k) for k in ("pws", "rots", "scales", "shs", "Rcw", "tcw", "twc")]
    args += [C.c_float(v) for v in (sc["fx"], sc["fy"], sc["cx"], sc["cy"], W, H)]
    if mom:
        args += [None, None, None]
    else:
        args += [p("gu"), p("gci"), p("gcol")]
    return args, T, (p("moments"), p("cinv2ds")) if mom else (None, None), p("gz") if depth else None


@pytest.mark.parametrize("mom", [False, True])
def test_pose_only_writes_nothing_and_is_reproducible(mom):
    from easygaussiansplatting_b200 import _lib
    lib = _lib.load()
    N, k3 = 20001, 16
    sc, st, up, W, H = _case(N, k3)
    keep = {}
    args, T, (mo, ci), gz = _abi_args(sc, W, H, up, mom, True, keep)
    inputs = {k: v.clone() for k, v in T.items()}
    wsb = lib.gsb_preprocess_backward_pose_workspace_bytes(N)
    ws = torch.full((wsb // 4 + 64,), float("nan"), device=DEV)
    gcam = torch.full((32,), 7.0, device=DEV)
    outs = []
    for _ in range(2):
        _lib.check(lib.gsb_preprocess_backward_pose(*args, None, None, None, None, mo, ci, None, None, gz,
                                                    gcam.data_ptr(), ws.data_ptr(), wsb, None), lib)
        torch.cuda.synchronize()
        outs.append(gcam.clone())
    assert torch.equal(bits(outs[0]), bits(outs[1]))                  # run to run: the same bits
    assert (gcam[15:] == 7.0).all() and torch.isnan(ws[wsb // 4:]).all()  # canaries
    for k, v in inputs.items():                                        # inputs untouched
        assert torch.equal(bits(T[k]), bits(v)), k
    # == the camera gradient of the full call, whose pre-filled outputs are all overwritten
    full = {k: torch.full(s, float("nan"), device=DEV) for k, s in (("pws", (N, 3)), ("shs", (N, 3 * k3)),
                                                                      ("scales", (N, 3)), ("rots", (N, 4)),
                                                                      ("dus", (N, 2)), ("dal", (N,)))}
    g2 = torch.full((15,), float("nan"), device=DEV)
    _lib.check(lib.gsb_preprocess_backward_pose(*args, *[full[k].data_ptr() for k in ("pws", "shs", "scales", "rots")],
                                                mo, ci, full["dus"].data_ptr() if mom else None,
                                                full["dal"].data_ptr() if mom else None, gz, g2.data_ptr(),
                                                ws.data_ptr(), wsb, None), lib)
    torch.cuda.synchronize()
    assert torch.equal(bits(g2), bits(outs[0][:15]))
    for k in ("pws", "shs", "scales", "rots") + (("dus", "dal") if mom else ()):
        assert not torch.isnan(full[k]).any(), k


def test_n0_gives_zeros():
    from easygaussiansplatting_b200 import _lib
    lib = _lib.load()
    sc, st, up, W, H = _case(1, 4)
    keep = {}
    args, T, _, _ = _abi_args(sc, W, H, up, False, False, keep)
    args[0] = 0
    g = torch.full((15,), float("nan"), device=DEV)
    assert lib.gsb_preprocess_backward_pose_workspace_bytes(0) == 0
    _lib.check(lib.gsb_preprocess_backward_pose(*args, None, None, None, None, None, None, None, None, None,
                                                g.data_ptr(), None, 0, None), lib)
    torch.cuda.synchronize()
    assert torch.equal(bits(g), torch.zeros(15, dtype=torch.int32, device=DEV))
    from easygaussiansplatting_b200 import ops
    e = lambda c: torch.empty((0, c), device=DEV)
    out = ops.preprocessB(e(3), e(4), e(3), e(12), t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]), sc["fx"], sc["fy"],
                          sc["cx"], sc["cy"], W, H, e(2), e(3), e(3), camera_grad=True)
    assert all(not x.any() for x in out[-1])


def test_bad_workspace_and_mixed_outputs_are_refused_before_launch():
    from easygaussiansplatting_b200 import _lib, ops
    lib = _lib.load()
    N = 1000
    sc, st, up, W, H = _case(N, 4)
    keep = {}
    args, T, (mo, ci), gz = _abi_args(sc, W, H, up, True, False, keep)
    wsb = lib.gsb_preprocess_backward_pose_workspace_bytes(N)
    ws = torch.zeros((wsb // 4 + 8,), device=DEV)
    g = torch.zeros((15,), device=DEV)
    o = {k: torch.zeros(s, device=DEV) for k, s in (("pws", (N, 3)), ("shs", (N, 12)), ("scales", (N, 3)),
                                                    ("rots", (N, 4)), ("dus", (N, 2)), ("dal", (N,)))}
    P = lambda k: o[k].data_ptr()
    idx = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())].index(
        "preprocess_backward")
    before = lib.gsb_profile_launches(idx)
    full = [P("pws"), P("shs"), P("scales"), P("rots"), mo, ci, P("dus"), P("dal"), None]
    bad = [
        (full, g.data_ptr(), ws.data_ptr() + 4, wsb, "misaligned"),
        (full, g.data_ptr(), ws.data_ptr(), wsb - 1, "too small"),
        (full, g.data_ptr(), None, wsb, "too small"),
        (full, None, ws.data_ptr(), wsb, "dloss_dcamera"),
        ([None, P("shs"), P("scales"), P("rots"), mo, ci, P("dus"), P("dal"), None], g.data_ptr(), ws.data_ptr(),
         wsb, "all set or all null"),
        ([P("pws"), None, P("scales"), P("rots"), mo, ci, P("dus"), P("dal"), None], g.data_ptr(), ws.data_ptr(),
         wsb, "all set or all null"),
        ([None, None, None, None, mo, ci, P("dus"), None, None], g.data_ptr(), ws.data_ptr(), wsb,
         "all set or all null"),
        ([None, None, None, None, mo, ci, None, P("dal"), None], g.data_ptr(), ws.data_ptr(), wsb,
         "all set or all null"),
    ]
    for outs, gp, wp, nb, msg in bad:
        rc = lib.gsb_preprocess_backward_pose(*args, *outs, gp, wp, nb, None)
        assert rc != 0 and msg in lib.gsb_last_error().decode(), (msg, lib.gsb_last_error())
    assert lib.gsb_profile_launches(idx) == before
    with pytest.raises(ValueError):
        _run(sc, W, H, up, False, False, pose_only=True)
    with pytest.raises(ValueError):
        _run(sc, W, H, up, True, False, camera_grad=True, compact=True)


# ---------------------------------------------------------------- autograd
class _Moments:
    """records the rasterizer backward's moment rows (and dL/dz) of one run and hands the same
    rows to the next: its atomics make them differ in the last bits from run to run"""

    def __init__(self, monkeypatch):
        from easygaussiansplatting_b200 import ops
        self.saved = None
        for name in ("splatB", "splatB_rgbd"):
            orig = getattr(ops, name)
            monkeypatch.setattr(ops, name, self._wrap(orig))

    def _wrap(self, orig):
        def f(*a, **kw):
            out = orig(*a, **kw)
            if self.saved is None:
                self.saved = [x.clone() for x in out] if isinstance(out, (list, tuple)) else out.clone()
            elif isinstance(out, (list, tuple)):
                out = [x.clone() for x in self.saved]
            else:
                out = self.saved.clone()
            return out
        return f


def _autograd(rgbd, sc, W, H, dl, dd, da, pose, need_map=True, chain_twc=False):
    from easygaussiansplatting_b200 import gsfunction as gf
    cam = gf.Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]))
    P = {k: t(sc[k]).requires_grad_(need_map) for k in ("pws", "shs", "scales", "rots")}
    al = t(sc["alphas"][:, None]).requires_grad_(need_map)
    us0 = torch.zeros((len(sc["pws"]), 2), device=DEV, requires_grad=need_map)
    gs = (P["pws"], P["shs"], al, P["scales"], P["rots"], us0)
    R = t(sc["Rcw"]).requires_grad_(bool(pose))
    tc = t(sc["tcw"]).requires_grad_(bool(pose))
    tw = -(R.t() @ tc) if chain_twc else t(sc["twc"]).requires_grad_(bool(pose))
    if pose is None:
        F = gf.GSFunctionFusedRGBD if rgbd else gf.GSFunctionFused
        outs = F.apply(*gs, cam)
    else:
        F = gf.GSFunctionFusedRGBDPose if rgbd else gf.GSFunctionFusedPose
        outs = F.apply(*gs, R, tc, tw, cam)
    if rgbd:
        ((outs[0] * dl).sum() + (outs[1] * dd).sum() + (outs[2] * da).sum()).backward()
    else:
        (outs[0] * dl).sum().backward()
    g = dict(pws=P["pws"].grad, shs=P["shs"].grad, alphas=al.grad, scales=P["scales"].grad, rots=P["rots"].grad,
             us=us0.grad)
    if pose:
        g.update(Rcw=R.grad, tcw=tc.grad, twc=None if chain_twc else tw.grad)
    return g, outs


def _oracle_from_moments(sc, W, H, moments, ddepths):
    """the pose oracle on the GPU's own splatB moment rows (fp64 conversion as the kernel does)"""
    st = opose.stages(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                      sc["fy"], sc["cx"], sc["cy"], W, H)
    from easygaussiansplatting_b200 import ops
    ci = ops.preprocess(*[t(sc[k]) for k in ("pws", "rots", "scales", "shs", "Rcw", "tcw", "twc")], sc["fx"],
                        sc["fy"], sc["cx"], sc["cy"], W, H)[1]
    gu, gci, gcol = _moment_grads(n(moments), n(ci))
    return opose.camera_grad(st, sc["pws"], sc["Rcw"], sc["fx"], sc["fy"], W, H, gu, gci, gcol,
                             None if ddepths is None else n(ddepths))


@pytest.mark.parametrize("rgbd", [False, True])
@pytest.mark.parametrize("sh_dim", [3, 48])
def test_autograd_pose_classes(monkeypatch, rgbd, sh_dim):
    N, W, H = 20000, 320, 240
    sc = gpu_scene(N, W, H, sh_dim, 21)
    rng = np.random.default_rng(5)
    dl = t(upstream_gradient(W, H, 3) * (3.0 * W * H))
    dd, da = t(rng.normal(size=(H, W)) * 0.3), t(rng.normal(size=(H, W)))
    rec = _Moments(monkeypatch)
    base, _ = _autograd(rgbd, sc, W, H, dl, dd, da, None)
    moments = rec.saved[0] if rgbd else rec.saved
    ddepths = rec.saved[1] if rgbd else None
    # the Gaussian gradients are those of GSFunctionFused(RGBD), bit for bit (same moment rows)
    g, _ = _autograd(rgbd, sc, W, H, dl, dd, da, True)
    for k in base:
        assert torch.equal(bits(g[k]), bits(base[k])), k
    # the camera gradient against the oracle on these moment rows
    ref = _oracle_from_moments(sc, W, H, moments, ddepths)
    got = np.concatenate([n(g["Rcw"]).reshape(-1), n(g["tcw"]), n(g["twc"])]).astype(np.float64)
    assert (np.abs(got - ref["grad"]) <= 1e-5 * ref["absum"]).all()
    assert np.abs(got[:12]).max() > 0 and (sh_dim == 3) == (not got[12:].any())
    # the camera alone: the pose-only kernel; the Gaussian leaves get nothing, the pose the same bits
    gp, _ = _autograd(rgbd, sc, W, H, dl, dd, da, True, need_map=False)
    for k in base:
        assert gp[k] is None, k
    for k in ("Rcw", "tcw", "twc"):
        assert torch.equal(bits(gp[k]), bits(g[k])), k
    # no camera gradient: exactly GSFunctionFused(RGBD)
    g0, _ = _autograd(rgbd, sc, W, H, dl, dd, da, False)
    for k in base:
        assert torch.equal(bits(g0[k]), bits(base[k])), k
    # twc = -Rcw^T tcw built in torch: autograd chains it into Rcw and tcw
    gc, _ = _autograd(rgbd, sc, W, H, dl, dd, da, True, need_map=False, chain_twc=True)
    R, tc = sc["Rcw"].astype(np.float64), sc["tcw"].astype(np.float64)
    wR, wt = opose.chain_twc(ref["grad"], R, tc)
    a = ref["absum"]
    tolR = 1e-5 * (a[:9].reshape(3, 3) + np.outer(np.abs(tc), a[12:])) + 1e-6 * np.abs(wR)
    tolt = 1e-5 * (a[9:12] + np.abs(R) @ a[12:]) + 1e-6 * np.abs(wt)
    assert (np.abs(n(gc["Rcw"]) - wR) <= tolR).all()
    assert (np.abs(n(gc["tcw"]) - wt) <= tolt).all()


def test_grad_exchange_is_refused():
    from easygaussiansplatting_b200 import gsfunction as gf
    sc = gpu_scene(100, 64, 48, 12, 3)
    cam = gf.Camera(64, 48, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]))
    cam.grad_exchange = object()
    args = [t(sc[k]) for k in ("pws", "shs")] + [t(sc["alphas"][:, None])] + [t(sc[k]) for k in ("scales", "rots")]
    args += [torch.zeros((100, 2), device=DEV), t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]), cam]
    with pytest.raises(ValueError):
        gf.GSFunctionFusedPose.apply(*args)


# ---------------------------------------------------------------- tracking
def _hat(xi):
    w, v = xi[:3], xi[3:]
    z = torch.zeros((), device=xi.device)
    return torch.stack([torch.stack([z, -w[2], w[1], v[0]]), torch.stack([w[2], z, -w[0], v[1]]),
                        torch.stack([-w[1], w[0], z, v[2]]), torch.stack([z, z, z, z])])


def test_rgbd_tracking_recovers_a_perturbed_pose():
    """the map is fixed and the pose of a frame is found by Adam on L1(image) + L1(depth), the
    pose an se(3) tangent through torch.matrix_exp; 1 degree and 2 cm off at the start"""
    from easygaussiansplatting_b200 import gsfunction as gf
    N, W, H = 20000, 640, 360
    sc = synthetic_scene(N, W, H, sh_dim=48, seed=4)
    sc["scales"] = (sc["scales"] * 3.0).astype(np.float32)  # smoother images: a wider basin
    a = 0.05
    Rt = torch.tensor([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]], device=DEV)
    tt = torch.tensor([0.05, -0.03, 0.1], device=DEV)
    cam = gf.Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], Rt, tt, -(Rt.t() @ tt))
    G = [t(sc[k]) for k in ("pws", "shs")] + [t(sc["alphas"][:, None])] + [t(sc[k]) for k in ("scales", "rots")]
    G.append(torch.zeros((N, 2), device=DEV))

    def render(R, tc):
        return gf.GSFunctionFusedRGBDPose.apply(*G, R, tc, -(R.t() @ tc), cam)

    with torch.no_grad():
        img_gt, dep_gt = [x.clone() for x in render(Rt, tt)[:2]]
    # start: 1 degree about an oblique axis, camera centre moved by 2 cm
    ax = torch.tensor([0.3, -0.8, 0.5], device=DEV)
    ax = ax / ax.norm()
    dR = torch.linalg.matrix_exp(_hat(torch.cat([ax * math.radians(1.0), torch.zeros(3, device=DEV)]))[:3, :3])
    R0 = dR @ Rt
    c_gt = -(Rt.t() @ tt)
    c0 = c_gt + torch.tensor([0.02, 0.0, 0.0], device=DEV)
    T0 = torch.eye(4, device=DEV)
    T0[:3, :3] = R0
    T0[:3, 3] = -(R0 @ c0)

    def errors(T):
        R, tc = T[:3, :3], T[:3, 3]
        c = -(R.t() @ tc)
        cosang = ((torch.trace(R @ Rt.t()) - 1) / 2).clamp(-1, 1)
        return torch.acos(cosang).item(), (c - c_gt).norm().item()

    e_rot0, e_t0 = errors(T0)
    assert abs(e_rot0 - math.radians(1.0)) < 1e-4 and abs(e_t0 - 0.02) < 1e-5
    xi = torch.zeros(6, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([xi], lr=2e-3)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=0.985)
    for _ in range(200):
        T = torch.linalg.matrix_exp(_hat(xi)) @ T0
        img, dep = render(T[:3, :3], T[:3, 3])[:2]
        loss = (img - img_gt).abs().mean() + (dep - dep_gt).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        sched.step()
    with torch.no_grad():
        e_rot, e_t = errors(torch.linalg.matrix_exp(_hat(xi)) @ T0)
    print("tracking: rotation %.3g -> %.3g rad, centre %.3g -> %.3g" % (e_rot0, e_rot, e_t0, e_t))
    assert e_rot < 0.1 * e_rot0 and e_t < 0.1 * e_t0, (e_rot, e_t)
