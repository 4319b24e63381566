"""GPU parity of the fused per-Gaussian path (gsb_preprocess_forward / _backward and
GSFunctionFused) against (a) the seven-operator path it replaces and (b) the CPU oracle /
reference-generated fixtures."""
import os

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from easygaussiansplatting_b200.scene import synthetic_scene, upstream_gradient

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
DEV = "cuda:0"


def t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).to(DEV)


def n(x):
    return x.detach().cpu().numpy()


def scene(N, W, H, sh_dim, seed):
    sc = synthetic_scene(N, W, H, sh_dim=sh_dim, seed=seed)
    rng = np.random.default_rng(seed + 3)
    idx = rng.choice(N, size=max(1, N // 50), replace=False)
    sc["pws"][idx, 2] = rng.uniform(-1.0, 0.19, len(idx)).astype(np.float32)
    wide = rng.choice(N, size=max(1, N // 50), replace=False)
    sc["pws"][wide, 0] *= 6.0
    if seed % 2 == 1:  # a general camera pose, so Rcw / tcw / twc really take part
        a, b = 0.15, -0.08
        Ry = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        Rx = np.array([[1, 0, 0], [0, np.cos(b), -np.sin(b)], [0, np.sin(b), np.cos(b)]])
        sc["Rcw"] = (Ry @ Rx).astype(np.float32)
        sc["tcw"] = np.array([0.3, -0.2, 0.4], np.float32)
        sc["twc"] = (-(sc["Rcw"].astype(np.float64).T @ sc["tcw"].astype(np.float64))).astype(np.float32)
        sc["rots"] = (sc["rots"] * rng.uniform(0.8, 1.25, (N, 1))).astype(np.float32)  # un-normalised q
    return sc


@pytest.mark.parametrize("N,sh_dim", [(1, 48), (129, 3), (5000, 12), (30000, 27), (100000, 48)])
def test_preprocess_equals_five_ops(N, sh_dim):
    import gsplatcu as g
    from easygaussiansplatting_b200 import ops
    W, H = 640, 360
    sc = scene(N, W, H, sh_dim, N)
    pws, rots, scales, shs = t(sc["pws"]), t(sc["rots"]), t(sc["scales"]), t(sc["shs"])
    Rcw, tcw, twc = t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"])
    us, pcs, depths = g.project(pws, Rcw, tcw, sc["fx"], sc["fy"], sc["cx"], sc["cy"], False)
    c3 = g.computeCov3D(rots, scales, depths, False)[0]
    c2 = g.computeCov2D(c3, pcs, Rcw, depths, sc["fx"], sc["fy"], W, H, False)[0]
    col = g.sh2Color(shs, pws, twc, False)[0]
    ci, areas = g.inverseCov2D(c2, depths, False)
    fus, fci, fcol, fd, far = ops.preprocess(pws, rots, scales, shs, Rcw, tcw, twc, sc["fx"], sc["fy"], sc["cx"],
                                             sc["cy"], W, H)
    assert torch.equal(fd < 0, depths < 0)
    assert torch.allclose(fus, us, rtol=1e-6, atol=1e-4) and torch.allclose(fd, depths, rtol=1e-6, atol=1e-6)
    assert torch.allclose(fcol, col, rtol=1e-5, atol=1e-5)
    assert torch.allclose(fci, ci, rtol=2e-4, atol=1e-6)
    assert (far != areas).float().mean().item() < 2e-3 and (far - areas).abs().max().item() <= 1
    assert not fus[fd < 0].any() and not fci[fd < 0].any() and not far[fd < 0].any()


def run_both(sc, W, H, seed=0):
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunction, GSFunctionFused
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]))
    dl = t(upstream_gradient(W, H, seed) * (3.0 * W * H))
    out = []
    for F in (GSFunction, GSFunctionFused):
        P = {k: t(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
        al = t(sc["alphas"][:, None]).requires_grad_()
        us0 = torch.zeros((len(sc["pws"]), 2), device=DEV, requires_grad=True)
        image, mask = F.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us0, cam)
        image.backward(dl)
        out.append(dict(image=image.detach(), mask=mask, pws=P["pws"].grad, shs=P["shs"].grad, alphas=al.grad,
                        scales=P["scales"].grad, rots=P["rots"].grad, us=us0.grad))
    return out


@pytest.mark.parametrize("N,W,H,sh_dim", [(20000, 320, 240, 48), (3000, 250, 130, 12), (500, 64, 64, 3),
                                          (4000, 979, 546, 27)])
def test_fused_function_matches_op_surface(N, W, H, sh_dim):
    a, b = run_both(scene(N, W, H, sh_dim, N + (N // 1000) % 2), W, H, N)  # 3000 -> rotated camera
    assert torch.equal(a["mask"], b["mask"])
    # a radius that flips by one between the two fp32 evaluation orders changes a tile list
    # but not the picture beyond the alpha' < 0.002 tail
    assert (a["image"] - b["image"]).abs().max().item() < 2e-3
    assert (a["image"] - b["image"]).abs().mean().item() < 1e-6
    for k in ("pws", "shs", "alphas", "scales", "rots", "us"):
        s = a[k].abs().max().item()
        e = (a[k] - b[k]).abs().max().item() / max(s, 1e-30)
        assert e < 2e-3, (k, e)
        em = (a[k] - b[k]).abs().mean().item() / max(a[k].abs().mean().item(), 1e-30)
        assert em < 1e-4, (k, em)


def test_fused_full_chain_golden_fixture():
    """params -> L1 loss -> parameter grads against backward_cpu.backward() (blend.npz)"""
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused
    bl = dict(np.load(os.path.join(G, "blend.npz")))
    fx, fy, cx, cy, W, H = bl["cam"]
    cam = Camera(int(W), int(H), fx, fy, cx, cy, t(bl["Rcw"]), t(bl["tcw"]), t(np.zeros(3, np.float32)))
    P = {k: t(bl[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    alphas = t(bl["alphas"][:, None]).requires_grad_()
    us = torch.zeros((len(bl["pws"]), 2), device=DEV, requires_grad=True)
    image, mask = GSFunctionFused.apply(P["pws"], P["shs"], alphas, P["scales"], P["rots"], us, cam)
    loss = torch.nn.functional.l1_loss(image, t(bl["image_gt"].transpose(2, 0, 1)))
    loss.backward()
    assert abs(loss.item() - float(bl["chain_loss"][0])) < 1e-5 and mask.all()
    for name, ref in (("rots", "chain_drots"), ("scales", "chain_dscales"), ("shs", "chain_dshs"),
                      ("pws", "chain_dpws")):
        e = np.abs(n(P[name].grad) - bl[ref]).max() / np.abs(bl[ref]).max()
        assert e < 1e-4, (name, e)
    e = np.abs(n(alphas.grad) - bl["chain_dalphas"]).max() / np.abs(bl["chain_dalphas"]).max()
    assert e < 1e-4, ("alphas", e)


def test_preprocess_backward_vs_oracle_chain():
    """gsb_preprocess_backward on random upstream grads vs the oracle's fp64 Jacobian chain"""
    from easygaussiansplatting_b200 import ops
    N, W, H, k3 = 40000, 640, 360, 16
    sc = scene(N, W, H, 3 * k3, 7)
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    us, pcs, depths, Ju = orc.project(sc["pws"], sc["Rcw"], sc["tcw"], sc["fx"], sc["fy"], sc["cx"], sc["cy"])
    d32 = f32(depths)
    c3, J3r, J3s = orc.compute_cov3d(sc["rots"], sc["scales"], d32)
    c2, J2c, J2p = orc.compute_cov2d(f32(c3), f32(pcs), sc["Rcw"], d32, sc["fx"], sc["fy"], W, H)
    col, Jcs, Jcp = orc.sh2color(sc["shs"], sc["pws"], sc["twc"])
    ci, areas, Jci = orc.inverse_cov2d(f32(c2), d32)
    rng = np.random.default_rng(0)
    gu = rng.normal(size=(N, 1, 2)).astype(np.float32); gci = rng.normal(size=(N, 1, 3)).astype(np.float32)
    gcol = rng.normal(size=(N, 1, 3)).astype(np.float32); gal = np.zeros((N, 1, 1), np.float32)
    keep = depths > 0
    gu[~keep] = 0; gci[~keep] = 0; gcol[~keep] = 0
    ref = orc.chain_backward(sc["Rcw"], gu, gci, gal, gcol, Ju, J3r, J3s, J2c, J2p, Jcs, Jcp, Jci)
    gpw, gsh, gs, gq = ops.preprocessB(t(sc["pws"]), t(sc["rots"]), t(sc["scales"]), t(sc["shs"]), t(sc["Rcw"]),
                                       t(sc["tcw"]), t(sc["twc"]), sc["fx"], sc["fy"], sc["cx"], sc["cy"], W, H,
                                       t(gu), t(gci), t(gcol))
    for got, name in ((gpw, "pws"), (gsh, "shs"), (gs, "scales"), (gq, "rots")):
        e = np.abs(n(got).astype(np.float64) - ref[name]).max() / np.abs(ref[name]).max()
        assert e < 2e-5, (name, e)


def test_record_cache_and_key_widths():
    """splatB reuses the forward's packed records only for untouched inputs; 32- and 64-bit key
    layouts (gsb_splat_render depth_key_max) give the same patch order."""
    import ctypes as C
    import gsplatcu as g
    from easygaussiansplatting_b200 import _lib, ops
    W, H, N = 320, 240, 20000
    sc = scene(N, W, H, 3, 21)
    us, ci, col, d, ar = ops.preprocess(t(sc["pws"]), t(sc["rots"]), t(sc["scales"]), t(sc["shs"]), t(sc["Rcw"]),
                                        t(sc["tcw"]), t(sc["twc"]), sc["fx"], sc["fy"], sc["cx"], sc["cy"], W, H)
    al = t(sc["alphas"])
    dl = t(upstream_gradient(W, H, 1) * (3.0 * W * H))
    out = g.splat(H, W, us, ci, al, d, col, ar)
    assert ops._cached_records(out[4], (us, ci, al, col)) is not None
    g1 = g.splatB(H, W, us, ci, al, d, col, out[1], out[2], out[3], out[4], dl)      # cached records
    # the handle rides on the tensor object: a copy (or any other tensor that happens to get the
    # same address later) has none
    assert ops._cached_records(out[4].clone(), (us, ci, al, col)) is None
    ops.forget_records(out[4])
    assert ops._cached_records(out[4], (us, ci, al, col)) is None
    g2 = g.splatB(H, W, us, ci, al, d, col, out[1], out[2], out[3], out[4], dl)      # re-packed
    for a, b in zip(g1, g2):
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-6 * a.abs().max().item())
    # an in-place edit of an input invalidates the cache entry
    out = g.splat(H, W, us, ci, al, d, col, ar)
    col.mul_(1.0)
    assert ops._cached_records(out[4], (us, ci, al, col)) is None
    # 64-bit reference key layout through the C ABI == the packed 32-bit layout
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    d2, ar2 = d.clone(), ar.clone()
    bin_bytes = lib.gsb_splat_bin_workspace_bytes(N)
    bin_ws = torch.empty(bin_bytes, dtype=torch.uint8, device=DEV)
    P, dk = C.c_int64(0), C.c_uint32(0)
    _lib.check(lib.gsb_splat_bin(H, W, N, us.data_ptr(), d2.data_ptr(), ar2.data_ptr(), bin_ws.data_ptr(), bin_bytes,
                                 C.byref(P), C.byref(dk), st), lib)
    P = int(P.value)
    assert P == out[4].numel() and 200 <= dk.value <= 20000
    ws_bytes = lib.gsb_splat_workspace_bytes(N, H, W, P)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
    img = torch.empty_like(out[0]); con = torch.empty_like(out[1]); ft = torch.empty_like(out[2])
    rg = torch.empty_like(out[3]); gs = torch.empty_like(out[4])
    _lib.check(lib.gsb_splat_render(H, W, N, P, 0xFFFFFFFF, us.data_ptr(), ci.data_ptr(), al.data_ptr(),
                                    d2.data_ptr(), col.data_ptr(), None, bin_ws.data_ptr(), ws.data_ptr(), ws_bytes,
                                    img.data_ptr(), con.data_ptr(), ft.data_ptr(), rg.data_ptr(), gs.data_ptr(), st),
               lib)
    assert torch.equal(gs, out[4]) and torch.equal(rg, out[3]) and torch.equal(img, out[0])


def test_fused_shortcuts_match_separate_passes():
    """preprocess(alphas=...) writes the same per-Gaussian records the pack pass builds, and
    preprocessB(moments=...) equals finalize + preprocessB on the four gradient tensors"""
    from easygaussiansplatting_b200 import ops
    W, H, N = 300, 200, 30000
    sc = scene(N, W, H, 48, 33)
    P = [t(sc[k]) for k in ("pws", "rots", "scales", "shs", "Rcw", "tcw", "twc")]
    cam = (sc["fx"], sc["fy"], sc["cx"], sc["cy"], W, H)
    al = t(sc["alphas"])
    plain = ops.preprocess(*P, *cam)
    withrec = ops.preprocess(*P, *cam, alphas=al)
    assert len(plain) == 5 and len(withrec) == 6 and tuple(withrec[5].shape) == (N, 12)
    for a, b in zip(plain, withrec):
        assert torch.equal(a, b)
    us, ci, col, d, ar = plain
    s1 = ops.splat(H, W, us, ci, al, d.clone(), col, ar.clone())
    s2 = ops.splat(H, W, us, ci, al, d.clone(), col, ar.clone(), records=withrec[5])
    for a, b in zip(s1, s2):
        assert torch.equal(a, b)
    dl = t(upstream_gradient(W, H, 5) * (3.0 * W * H))
    g4 = ops.splatB(H, W, us, ci, al, d, col, s2[1], s2[2], s2[3], s2[4], dl)
    m = ops.splatB(H, W, us, ci, al, d, col, s2[1], s2[2], s2[3], s2[4], dl, moments_only=True)
    assert tuple(m.shape) == (N, 9)
    a = ops.preprocessB(*P, *cam, g4[0], g4[1], g4[3])
    b = ops.preprocessB(*P, *cam, None, None, None, moments=m, cinv2ds=ci)
    assert len(a) == 4 and len(b) == 6
    # (two backward launches accumulate their moment rows with float atomics in different orders)
    for x, y in zip(a, b[:4]):
        assert float((x - y).abs().max() / x.abs().max()) <= 1e-5
    assert float((b[4] - g4[0].reshape(N, 2)).abs().max() / g4[0].abs().max()) <= 1e-5
    assert float((b[5] - g4[2].reshape(N)).abs().max() / g4[2].abs().max()) <= 1e-5
    with pytest.raises(RuntimeError, match="go together"):
        _lib_call_preprocess_with_records_only(ops, P, cam, N)


def _lib_call_preprocess_with_records_only(ops, P, cam, N):
    from easygaussiansplatting_b200 import _lib
    lib = _lib.load()
    o = [torch.empty((N, k), device=DEV) for k in (2, 3, 3)] + [torch.empty(N, device=DEV),
                                                                torch.empty((N, 2), dtype=torch.int32, device=DEV)]
    rec = torch.empty((N, 12), device=DEV)
    _lib.check(lib.gsb_preprocess_forward(N, 16, *[x.data_ptr() for x in P], *[float(c) for c in cam],
                                          *[x.data_ptr() for x in o], None, rec.data_ptr(), None), lib)


@pytest.mark.parametrize("N,W,H", [(20000, 320, 240), (400, 1000, 700), (3000, 979, 546)])
def test_capacity_path_equals_exact_path(N, W, H):
    """gsb_splat_forward (sort sized from the previous frame, status read after everything is
    enqueued) gives bit-identical outputs to gsb_splat_bin + gsb_splat_render; a frame that outgrows
    its bounds -- patch count or depth-key width -- is redone the exact way."""
    from easygaussiansplatting_b200 import ops
    sc = scene(N, W, H, 12, 5)
    args = (t(sc["pws"]), t(sc["rots"]), t(sc["scales"]), t(sc["shs"]), t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]),
            sc["fx"], sc["fy"], sc["cx"], sc["cy"], W, H)
    al = t(sc["alphas"])

    def run(capacity):
        u, ci, col, dep, ar = ops.preprocess(*args)
        return ops.splat(H, W, u, ci, al, dep, col, ar, capacity=capacity), dep, ar

    ops._CAPACITY.clear()
    exact, dep0, ar0 = run(False)
    first, _, _ = run(True)   # learns the capacities (exact path)
    key = (0, H, W, N)
    assert key in ops._CAPACITY
    cap, dep1, ar1 = run(True)  # capacity path
    assert ops._CAPACITY[key][0] >= cap[4].numel()
    for a, b, c in zip(exact, first, cap):
        assert torch.equal(a, b) and torch.equal(a, c)
    assert torch.equal(dep0, dep1) and torch.equal(ar0, ar1)
    P = exact[4].numel()

    def poison():
        """fill the caching allocator's pool with ids far outside [0, N): after an overflow the key / id
        arrays have holes the kernels never wrote, and nothing may be gathered through them"""
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        x = torch.full((64 << 20,), 0x7f7f7f7f, dtype=torch.int32, device=DEV)
        torch.cuda.synchronize()
        del x

    poison()
    ops._CAPACITY[key] = (max(1, P // 3), ops._CAPACITY[key][1])  # too few patches
    small, _, _ = run(True)
    torch.cuda.synchronize()
    poison()
    ops._CAPACITY[key] = (2 * P + 10, 3)                          # depth keys wider than planned
    narrow, _, _ = run(True)
    torch.cuda.synchronize()
    for a, b, c in zip(exact, small, narrow):
        assert torch.equal(a, b) and torch.equal(a, c)
    assert ops._CAPACITY[key][0] >= P  # relearnt


@pytest.mark.parametrize("N,W,H,sh_dim,V", [(20000, 320, 240, 48, 3), (3000, 200, 120, 12, 1), (500, 64, 64, 3, 2)])
def test_factorised_multi_view_step_matches_autograd_accumulation(N, W, H, sh_dim, V):
    """parallel.MultiViewStep (per view: 11 small gradient floats accumulated + dL/dcolor kept; one
    expansion dL/dsh = sum_v Y(dir_v) (x) dL/dcolor_v at the end) against the plain accumulation
    of GSFunctionFused's gradients over the same V views.  Agreement is to rounding, not bitwise:
    the rasterizer backward's atomics make two runs of the same view differ in the last bits."""
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused
    from easygaussiansplatting_b200.parallel import MultiViewStep
    from easygaussiansplatting_b200.scene import ring_camera
    sc = scene(N, W, H, sh_dim, 4)
    P = {k: t(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    al = t(sc["alphas"][:, None]).requires_grad_()
    us0 = torch.zeros((N, 2), device=DEV, requires_grad=True)
    cams, dls = [], []
    for v in range(V):
        Rcw, tcw, twc = ring_camera(v, 8) if V > 1 else (sc["Rcw"], sc["tcw"], sc["twc"])
        cams.append(Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(Rcw), t(tcw), t(twc)))
        dls.append(t(upstream_gradient(W, H, v) * (3.0 * W * H)))
    for cam, dl in zip(cams, dls):
        image, _ = GSFunctionFused.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us0, cam)
        image.backward(dl)
    mv = MultiViewStep(P["pws"].detach(), P["rots"].detach(), P["scales"].detach(), P["shs"].detach(), al.detach())
    for cam, dl in zip(cams, dls):
        img, ctx = mv.render(cam)
        mv.backward(ctx, dl)
    g = mv.reduce()
    assert g["bytes_per_rank"] == 4 * N * (11 + 3 * V)
    for name, want in (("dpws", P["pws"].grad), ("dshs", P["shs"].grad), ("dscales", P["scales"].grad),
                       ("drots", P["rots"].grad), ("dalphas", al.grad.reshape(-1))):
        got = g[name].reshape(want.shape)
        err = float((got - want).abs().max() / want.abs().max().clamp_min(1e-30))
        assert err <= 2e-6, (name, err)


def test_graphed_step_matches_eager_and_detects_overflow():
    """graphed.GraphedFusedStep (forward and backward replayed as CUDA graphs over static buffers,
    capacity-based rasterizer, lazily checked status) against the eager fused autograd path; new
    parameter values written in place are seen by the next replay; a frame that outgrows the
    captured capacity raises CapacityError."""
    from easygaussiansplatting_b200.graphed import CapacityError, GraphedFusedStep
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused
    N, W, H, sh_dim = 20000, 320, 240, 12
    sc = scene(N, W, H, sh_dim, 6)
    P = {k: t(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    al = t(sc["alphas"][:, None]).requires_grad_()
    us0 = torch.zeros((N, 2), device=DEV, requires_grad=True)
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]))
    dl = t(upstream_gradient(W, H, 1) * (3.0 * W * H))
    # the graph's static buffers come out of a pool full of out-of-range ids (see the overflow below)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    junk = torch.full((64 << 20,), 0x7f7f7f7f, dtype=torch.int32, device=DEV)
    torch.cuda.synchronize()
    del junk
    torch.cuda.empty_cache()  # (the capture allocates from its own pool: hand the dirty pages back to the driver)
    step = GraphedFusedStep(P["pws"], P["shs"], al, P["scales"], P["rots"], cam)

    def eager():
        for p in list(P.values()) + [al]:
            p.grad = None
        image, _ = GSFunctionFused.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us0, cam)
        image.backward(dl)
        return image.detach()

    for rep in range(2):
        want = eager()
        img = step.forward()
        assert torch.equal(img, want)
        step.dloss_dimage.copy_(dl)
        g = step.backward()
        for name, ref in (("dpws", P["pws"].grad), ("dshs", P["shs"].grad), ("dscales", P["scales"].grad),
                          ("drots", P["rots"].grad), ("dalphas", al.grad.reshape(-1))):
            err = float((g[name].reshape(ref.shape) - ref).abs().max() / ref.abs().max().clamp_min(1e-30))
            assert err <= 2e-6, (name, err)
        with torch.no_grad():  # an in-place parameter update is picked up by the next replay
            P["pws"].add_(0.01 * torch.randn_like(P["pws"]))
            P["scales"].mul_(1.05)
    # blow the scene up so that the patch count exceeds the captured capacity
    with torch.no_grad():
        P["scales"].mul_(4.0)
    step.forward()
    torch.cuda.synchronize()  # the overflowing replay itself must be memory-safe
    with pytest.raises(CapacityError):
        step.backward()
    step.recapture()
    assert torch.equal(step.forward(), eager())
