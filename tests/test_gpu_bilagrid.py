"""The bilateral-grid kernels on the GPU (DESIGN 3.20) against the fp64 oracle
(oracle/bilagrid_oracle.py): the slice and both gradients at tile and cell edges, at 1920 x 1080,
at other grid sizes, for batches with a repeated grid and inputs outside [0, 1]; the TV; the
identity grid; the module chain against the same chain through F.grid_sample; and a fit to views
whose colours were shifted per view."""
import numpy as np
import pytest
import torch

from oracle import bilagrid_oracle as bo

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _case(M, L, Y, X, B, H, W, seed, lo=0.0, hi=1.0, spread=0.3):
    rng = np.random.default_rng(seed)
    eye = np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], dtype=np.float32).reshape(1, 12, 1, 1, 1)
    grids = (eye + spread * rng.standard_normal((M, 12, L, Y, X))).astype(np.float32)
    rgb = rng.uniform(lo, hi, (B, 3, H, W)).astype(np.float32)
    dout = rng.standard_normal((B, 3, H, W)).astype(np.float32)
    return grids, rgb, dout


CASES = [  # H, W, X, Y, L, ids, rgb range
    (37, 53, 16, 16, 8, [0], (0.0, 1.0)),
    (1080, 1920, 16, 16, 8, [1], (0.0, 1.0)),
    (64, 96, 5, 3, 1, [0], (-0.2, 1.2)),
    (50, 70, 1, 7, 4, [2], (0.0, 1.0)),
    (29, 31, 64, 64, 64, [1], (0.0, 1.0)),     # cells narrower than a pixel; 64 levels
    (120, 160, 12, 9, 5, [1, 0, 1], (-0.3, 1.3)),  # a batch with a repeated grid
    (1, 1, 2, 2, 2, [0], (0.0, 1.0)),
]


@pytest.mark.parametrize("H,W,X,Y,L,ids,rng_", CASES, ids=["%dx%d-X%dY%dL%d-B%d" % (c[1], c[0], *c[2:5], len(c[5]))
                                                            for c in CASES])
def test_slice_and_backward_match_the_oracle(H, W, X, Y, L, ids, rng_):
    from easygaussiansplatting_b200 import ops
    grids, rgb, dout = _case(3, L, Y, X, len(ids), H, W, seed=H + W + X + L, lo=rng_[0], hi=rng_[1])
    ref = bo.slice_grids(grids, rgb, ids, dout)
    g, r, d = (torch.from_numpy(a).to(DEV) for a in (grids, rgb, dout))
    out = ops.bilagrid_slice(g, r, ids)
    drgb, dgrids = ops.bilagrid_sliceB(g, r, ids, d)
    np.testing.assert_allclose(out.cpu().numpy(), ref["out"], rtol=0, atol=1e-5)
    ok = ~ref["ambiguous"][:, None].repeat(3, axis=1)
    # the guidance term is (L - 1) dL/dout . (A1 - A0) [rgb, 1]: the fp32 rounding of A1 - A0 is
    # scaled by (L - 1) sum|dL/dout| sum|[rgb, 1]|
    cond = (L - 1) * np.abs(dout).sum(1, keepdims=True) * (np.abs(rgb).sum(1, keepdims=True) + 1) * np.abs(grids).max()
    tol = np.broadcast_to(1e-5 + 1e-6 * cond, rgb.shape)
    err = np.abs(drgb.cpu().numpy() - ref["drgb"])
    assert (err[ok] <= tol[ok]).all(), (err[ok].max(), (err[ok] / tol[ok]).max())
    err = np.abs(dgrids.cpu().numpy() - ref["dgrids"])
    # summation order against the sum of |terms|, and the fp32 rounding of the pixel coordinates
    bound = 2e-5 * ref["dgrids_cond"] + 1e-6 * ref["dgrids_cond_t"] + 1e-6
    assert (err <= bound).all(), (err.max(), np.unravel_index(np.argmax(err - bound), err.shape))
    # a single image with one index gives the batch item's planes
    assert torch.equal(ops.bilagrid_slice(g, r[0], ids[0]), out[0])


def test_backward_adds_into_a_given_gradient():
    from easygaussiansplatting_b200 import ops
    grids, rgb, dout = _case(2, 8, 16, 16, 1, 40, 60, seed=11)
    g, r, d = (torch.from_numpy(a).to(DEV) for a in (grids, rgb, dout))
    _, first = ops.bilagrid_sliceB(g, r, [1], d)
    acc = first.clone()
    ops.bilagrid_sliceB(g, r, [1], d, dloss_dgrids=acc)
    torch.testing.assert_close(acc, 2 * first, rtol=1e-6, atol=1e-7)
    with pytest.raises(TypeError, match="CUDA tensor"):
        ops.bilagrid_slice(g, r, torch.tensor([0], device=DEV))
    with pytest.raises(ValueError, match=r"\[0, 2\)"):
        ops.bilagrid_slice(g, r, [2])
    with pytest.raises(ValueError, match="image ids for a batch"):
        ops.bilagrid_slice(g, r, [0, 1])
    assert torch.equal(ops.bilagrid_slice(g, r, torch.tensor([1])), ops.bilagrid_slice(g, r, [1]))


@pytest.mark.parametrize("shape", [(300, 12, 8, 16, 16), (2, 12, 1, 3, 5), (3, 12, 4, 1, 1), (1, 12, 1, 1, 1),
                                   (1, 12, 64, 64, 64)])
def test_total_variation_matches_the_oracle(shape):
    from easygaussiansplatting_b200 import ops
    g = (np.random.default_rng(len(shape) + shape[0]).standard_normal(shape) * 0.1).astype(np.float32)
    tv_ref, grad_ref = bo.total_variation(g)
    t = torch.from_numpy(g).to(DEV)
    tv, grad = ops.bilagrid_tv(t)
    assert abs(tv.item() - tv_ref) <= 1e-6 * max(abs(tv_ref), 1e-30), (tv.item(), tv_ref)
    np.testing.assert_allclose(grad.cpu().numpy(), grad_ref, rtol=0, atol=1e-6 * max(np.abs(grad_ref).max(), 1e-30))
    tv2, none = ops.bilagrid_tv(t, want_grad=False)
    assert none is None and torch.equal(tv, tv2)  # the value is summed in a fixed order


def test_identity_grid_reproduces_the_image():
    from easygaussiansplatting_b200.bilagrid import BilateralGrid
    bil = BilateralGrid(4, device=DEV)
    rgb = torch.from_numpy(_case(1, 1, 1, 1, 2, 257, 381, seed=2, lo=-0.5, hi=1.5)[1]).to(DEV)
    out = bil(rgb, [3, 3])
    ulp = (out.view(torch.int32).long() - rgb.view(torch.int32).long()).abs().max().item()
    assert ulp <= 1, ulp


def _fused_scene(W=160, H=96, N=2000):
    from easygaussiansplatting_b200.gsfunction import Camera
    from easygaussiansplatting_b200.scene import synthetic_scene
    sc = synthetic_scene(N, W, H, sh_dim=48, seed=0)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], T(sc["Rcw"]), T(sc["tcw"]), T(sc["twc"]))
    return sc, cam, T, W, H


def test_module_chain_matches_the_grid_sample_chain():
    from easygaussiansplatting_b200.bilagrid import BilateralGrid
    from easygaussiansplatting_b200.gsfunction import GSFunctionFused
    from easygaussiansplatting_b200.loss import gau_loss
    sc, cam, T, W, H = _fused_scene()
    rng = np.random.default_rng(4)
    gt = T(rng.uniform(0, 1, (3, H, W)).astype(np.float32))
    bil = BilateralGrid(3, device=DEV)
    with torch.no_grad():
        bil.grids.add_(torch.from_numpy((0.2 * rng.standard_normal(bil.grids.shape)).astype(np.float32)).to(DEV))
    grids_t = bil.grids.detach().clone().requires_grad_()
    grads = []
    for use_kernel in (True, False):
        P = {k: T(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
        alphas = T(sc["alphas"][:, None]).requires_grad_()
        us = torch.zeros((sc["pws"].shape[0], 2), device=DEV, requires_grad=True)
        image, _ = GSFunctionFused.apply(P["pws"], P["shs"], alphas, P["scales"], P["rots"], us, cam)
        if use_kernel:
            loss = gau_loss(bil(image, 1), gt) + 10.0 * bil.tv_loss()
            G = bil.grids
        else:
            tv = sum((grids_t.diff(dim=a) ** 2).mean() for a in (2, 3, 4))
            loss = gau_loss(bo.torch_slice(grids_t, image, 1), gt) + 10.0 * tv
            G = grids_t
        loss.backward()
        grads.append([P["pws"].grad, P["shs"].grad, P["scales"].grad, P["rots"].grad, alphas.grad, G.grad])
    for name, a, b in zip(("pws", "shs", "scales", "rots", "alphas", "grids"), *grads):
        e = (a - b).abs().max().item() / b.abs().max().item()
        assert e < 1e-4, (name, e)


def test_grid_per_view_fits_colour_shifted_views_better():
    """views of a hidden scene with per-view gains (0.6 to 1.4 per channel) and offsets: a grid per
    view ends at a lower L1 against them than the same steps without grids"""
    from easygaussiansplatting_b200.bilagrid import BilateralGrid
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused
    from easygaussiansplatting_b200.scene import ring_camera, synthetic_scene
    n, views, iters, W, H = 4000, 4, 160, 160, 120
    gt = synthetic_scene(n, W, H, sh_dim=48, seed=0)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    cams = [Camera(W, H, gt["fx"], gt["fy"], gt["cx"], gt["cy"], *(T(a) for a in ring_camera(k, views, radius=0.3)))
            for k in range(views)]
    rng = np.random.default_rng(12)
    gains = T(rng.uniform(0.6, 1.4, (views, 3, 1, 1)).astype(np.float32))
    offsets = T(rng.uniform(-0.05, 0.05, (views, 3, 1, 1)).astype(np.float32))
    us0 = torch.zeros((n, 2), device=DEV)
    with torch.no_grad():
        targets = [GSFunctionFused.apply(T(gt["pws"]), T(gt["shs"]), T(gt["alphas"][:, None]), T(gt["scales"]),
                                         T(gt["rots"]), us0, c)[0] * gains[k] + offsets[k] for k, c in enumerate(cams)]

    def run(with_grid):
        torch.manual_seed(0)
        r = np.random.default_rng(1)
        pws = torch.nn.Parameter(T(gt["pws"] + r.normal(scale=0.01, size=gt["pws"].shape).astype(np.float32)))
        low = torch.nn.Parameter(torch.zeros((n, 3), device=DEV))
        high = torch.nn.Parameter(torch.full((n, 45), 0.001, device=DEV))
        alphas_raw = torch.nn.Parameter(torch.zeros((n, 1), device=DEV))
        scales_raw = torch.nn.Parameter(torch.log(T(gt["scales"] * 1.3)))
        rots_raw = torch.nn.Parameter(T(gt["rots"]))
        opt = torch.optim.Adam([{"params": [pws], "lr": 0.001}, {"params": [low], "lr": 0.02},
                                {"params": [high], "lr": 0.001}, {"params": [alphas_raw], "lr": 0.05},
                                {"params": [scales_raw], "lr": 0.005}, {"params": [rots_raw], "lr": 0.001}], eps=1e-15)
        bil = BilateralGrid(views, grid_X=4, grid_Y=4, grid_L=4, device=DEV) if with_grid else None
        # a larger step than gsplat's 2e-3: the run is 160 steps, not 30k
        gopt = torch.optim.Adam(bil.parameters(), lr=1e-2) if with_grid else None
        us = torch.zeros((n, 2), device=DEV, requires_grad=True)
        losses = []
        for it in range(iters):
            k = it % views
            image, _ = GSFunctionFused.apply(pws, torch.cat((low, high), 1), torch.sigmoid(alphas_raw),
                                             torch.exp(scales_raw), torch.nn.functional.normalize(rots_raw), us, cams[k])
            if with_grid:
                image = bil(image, k)
            loss = torch.nn.functional.l1_loss(image, targets[k])
            if with_grid:
                loss = loss + 10.0 * bil.tv_loss()
            opt.zero_grad(set_to_none=True)
            if with_grid:
                gopt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            if with_grid:
                gopt.step()
            losses.append(torch.nn.functional.l1_loss(image.detach(), targets[k]).item())
        return float(np.mean(losses[-views:]))

    plain, graded = run(False), run(True)
    assert graded < 0.9 * plain, (graded, plain)
