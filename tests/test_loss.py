"""Training loss (SURVEY 8f row N2).  CPU: the oracle's gau_loss against the fixture produced by
the reference's own gsplat/pytorch_ssim.py (tests/golden/make_golden_loss.py).  GPU: the fused
kernels against the oracle, the fixture, and a torch transcription of pytorch_ssim.py:26-67."""
import os

import numpy as np
import pytest
import torch

from oracle import oracle as orc

G = os.path.join(os.path.dirname(__file__), "golden", "loss.npz")


def test_oracle_matches_reference_fixture():
    d = dict(np.load(G))
    for k in "ab":
        r = orc.gau_loss(d["img_" + k], d["gt_" + k])
        assert abs(r["loss"] - float(d["loss_" + k])) < 2e-6          # reference runs in float32
        ref = d["grad_" + k]
        assert np.abs(r["dloss_dimage"] - ref).max() / np.abs(ref).max() < 2e-4
    w = orc.ssim_window()
    assert abs(w.sum() - 1) < 1e-6 and w.argmax() == 5 and np.allclose(w, w[::-1])


def test_oracle_identical_images_and_lambda():
    img = np.random.default_rng(0).uniform(0, 1, (3, 20, 24)).astype(np.float32)
    r = orc.gau_loss(img, img.copy())
    assert abs(r["l1"]) < 1e-12 and abs(r["ssim"] - 1) < 1e-9 and abs(r["loss"]) < 1e-9
    gt = np.clip(img + 0.1, 0, 1).astype(np.float32)
    a, b = orc.gau_loss(img, gt, 0.0), orc.gau_loss(img, gt, 1.0)
    assert abs(a["loss"] - a["l1"]) < 1e-12 and abs(b["loss"] - (1 - b["ssim"])) < 1e-12


def test_oracle_gradient_is_numerical_derivative():
    rng = np.random.default_rng(3)
    img = rng.uniform(0.2, 0.8, (3, 14, 13)).astype(np.float32)
    gt = rng.uniform(0.2, 0.8, (3, 14, 13)).astype(np.float32)
    r = orc.gau_loss(img, gt)
    for (c, y, x) in [(0, 0, 0), (1, 7, 6), (2, 13, 12), (0, 5, 11)]:
        h = np.float32(2.0 ** -10)  # exactly representable step
        p, m = img.copy(), img.copy()
        p[c, y, x] += h; m[c, y, x] -= h
        num = (orc.gau_loss(p, gt, want_grad=False)["loss"] - orc.gau_loss(m, gt, want_grad=False)["loss"]) / (
            float(p[c, y, x]) - float(m[c, y, x]))
        assert abs(num - r["dloss_dimage"][c, y, x]) < 2e-6 + 1e-3 * abs(num)


def _torch_gau_loss(image, gt, lam=0.2):
    """transcription of pytorch_ssim.py:26-67 for CUDA tensors (the tests never import the reference)"""
    import torch.nn.functional as F
    g = torch.tensor([np.exp(-(x - 5) ** 2 / float(2 * 1.5 ** 2)) for x in range(11)], dtype=torch.float32)
    g = (g / g.sum()).unsqueeze(1)
    win = g.mm(g.t()).float().unsqueeze(0).unsqueeze(0).expand(3, 1, 11, 11).contiguous().to(image.device)
    mu1 = F.conv2d(image, win, padding=5, groups=3); mu2 = F.conv2d(gt, win, padding=5, groups=3)
    s11 = F.conv2d(image * image, win, padding=5, groups=3) - mu1.pow(2)
    s22 = F.conv2d(gt * gt, win, padding=5, groups=3) - mu2.pow(2)
    s12 = F.conv2d(image * gt, win, padding=5, groups=3) - mu1 * mu2
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    ssim = ((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1.pow(2) + mu2.pow(2) + C1) * (s11 + s22 + C2))
    return (1 - lam) * torch.abs(image - gt).mean() + lam * (1 - ssim.mean())


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(37, 53), (16, 16), (128, 96), (1080, 1920),
                                 (1, 1), (2, 300), (300, 2), (15, 31)])   # strips narrower than a warp
def test_gpu_gau_loss_vs_oracle(H, W):
    from easygaussiansplatting_b200.loss import gau_loss, gau_loss_with_grad
    rng = np.random.default_rng(H * 1000 + W)
    yy, xx = np.mgrid[0:H, 0:W]
    base = np.stack([0.5 + 0.4 * np.sin(xx / 9.0 + c) * np.cos(yy / 6.0 - c) for c in range(3)])
    img = np.clip(base + rng.normal(scale=0.08, size=base.shape), -0.2, 1.3).astype(np.float32)
    gt = np.clip(base + rng.normal(scale=0.02, size=base.shape), 0, 1).astype(np.float32)
    ref = orc.gau_loss(img, gt)
    ti = torch.from_numpy(img).cuda().requires_grad_(); tg = torch.from_numpy(gt).cuda()
    loss = gau_loss(ti, tg)
    loss.backward()
    assert abs(loss.item() - ref["loss"]) < 2e-6
    got = ti.grad.cpu().numpy().astype(np.float64)
    e = np.abs(got - ref["dloss_dimage"]).max() / np.abs(ref["dloss_dimage"]).max()
    assert e < 3e-4, e   # float32 E[x^2] - mu^2 cancellation, the same formulation as the reference
    # the torch transcription of the reference agrees too
    t2 = torch.from_numpy(img).cuda().requires_grad_()
    l2 = _torch_gau_loss(t2, tg)
    l2.backward()
    assert abs(l2.item() - loss.item()) < 2e-6
    assert (t2.grad - ti.grad).abs().max().item() / t2.grad.abs().max().item() < 3e-4
    # loss only (no gradient buffer) and scaling through autograd
    lo, g = gau_loss_with_grad(tg + 0.05, tg, 0.2, want_grad=False)
    assert g is None and lo.item() > 0
    t3 = torch.from_numpy(img).cuda().requires_grad_()
    (3.0 * gau_loss(t3, tg)).backward()
    assert torch.allclose(t3.grad, 3.0 * ti.grad, rtol=1e-6, atol=0)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["img", "gt"])
def test_gpu_gau_loss_unaligned_view_is_bit_identical(which):
    """W % 4 == 0, but the image starts one float into its storage: the row kernels take their
    scalar loads instead of the 16-byte ones, with the same arithmetic -- loss and gradient are
    bit-identical to the aligned call"""
    from easygaussiansplatting_b200.loss import gau_loss_with_grad
    H, W = 45, 136
    rng = np.random.default_rng(5)
    img = torch.from_numpy(rng.uniform(0, 1, (3, H, W)).astype(np.float32)).cuda()
    gt = torch.from_numpy(rng.uniform(0, 1, (3, H, W)).astype(np.float32)).cuda()
    la, ga = gau_loss_with_grad(img, gt, 0.2)
    buf = torch.empty(3 * H * W + 1, device="cuda")
    view = buf[1:].view(3, H, W)
    view.copy_(img if which == "img" else gt)
    assert view.is_contiguous() and view.data_ptr() % 16 == 4
    lb, gb = gau_loss_with_grad(view, gt, 0.2) if which == "img" else gau_loss_with_grad(img, view, 0.2)
    assert torch.equal(la, lb) and torch.equal(ga, gb)


def _patched_pair(H, W, corners, rng, P=64):
    """img, gt [3, H, W] on the GPU: zero except P x P patches of random content at `corners`"""
    img = torch.zeros((3, H, W), device="cuda")
    gt = torch.zeros((3, H, W), device="cuda")
    for (y, x) in corners:
        a = rng.uniform(0, 1, (3, P, P)).astype(np.float32)
        b = np.clip(a + rng.normal(scale=0.1, size=a.shape), 0, 1).astype(np.float32)
        img[:, y:y + P, x:x + P] = torch.from_numpy(a).cuda()
        gt[:, y:y + P, x:x + P] = torch.from_numpy(b).cuda()
    return img, gt


@pytest.mark.gpu
def test_gpu_gau_loss_at_and_above_the_tiled_bound():
    """The loss at two sizes next to the switch between the row kernels and the tiled kernels
    (H W < 2^31 / 9, about 238.6 Mpixels): 14563 x 16384 is the largest row-path image of that
    width (vector loads), 14567 x 16381 is just above it and takes the tiled kernels with ragged
    tiles on both axes (W % 32 = 29, H % 16 = 7) and map offsets past 2^31 in channel 2.

    img = gt = 0 except a few 64 x 64 patches (image corners -- the largest offsets of every
    channel -- and across tile / CTA / strip boundaries).  With zero padding no pixel sees content
    more than 10 px away, so inside a crop with >= 20 zero pixels (or the image edge) around its
    patch the gradient is the oracle's gradient of the crop times n_crop / n_full, and it is
    exactly 0 everywhere else."""
    from easygaussiansplatting_b200.loss import gau_loss_with_grad
    need = 18 << 30
    free, total = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB of %.1f GB free" % (need / 2**30, free / 2**30,
                                                                                    total / 2**30))
    # the kernels' fp32 SSIM of an all-zero neighbourhood (C1 C2 / (C1 C2) need not round to 1)
    z = torch.zeros((3, 32, 32), device="cuda")
    ssim0 = 1.0 - float(gau_loss_with_grad(z, z, 1.0, want_grad=False)[0])
    lam, P, M = 0.2, 64, 20
    torch.cuda.reset_peak_memory_stats()
    for H, W in ((14563, 16384), (14567, 16381)):
        rng = np.random.default_rng(H)
        corners = [(0, 0), (H - P, W - P), (0, W - P), (H - P, 0),
                   (H // 2 - 37, 128 * 60 - 29),           # row path: CTA boundary (128 columns)
                   (16 * 401 - 31, 32 * 223 - 17),         # tiled: corners of 32 x 16 tiles
                   (7 * H // 8 + 3, W // 3 + 5)]
        img, gt = _patched_pair(H, W, corners, rng, P)
        loss, grad = gau_loss_with_grad(img, gt, lam)
        n_full = 3.0 * H * W
        l1_sum = ss_sum = 0.0
        n_crops = 0.0
        for (y, x) in corners:
            y0, y1, x0, x1 = max(0, y - M), min(H, y + P + M), max(0, x - M), min(W, x + P + M)
            ci = img[:, y0:y1, x0:x1].cpu().numpy()
            cg = gt[:, y0:y1, x0:x1].cpu().numpy()
            ref = orc.gau_loss(ci, cg, lam)
            n_crop = float(ci.size)
            want = ref["dloss_dimage"] * (n_crop / n_full)
            got = grad[:, y0:y1, x0:x1].cpu().numpy().astype(np.float64)
            e = np.abs(got - want).max() / np.abs(want).max()
            assert e < 3e-4, (H, W, y, x, e)   # the bound of test_gpu_gau_loss_vs_oracle
            l1_sum += ref["l1"] * n_crop
            ss_sum += ref["ssim"] * n_crop
            n_crops += n_crop
            grad[:, y0:y1, x0:x1] = 0
        assert not bool(grad.any()), "gradient outside the patch crops (%d x %d)" % (H, W)
        # the background counts at the kernels' SSIM of zero.  Tolerance: inside the crops the
        # oracle's zero pixels have SSIM exactly 1 where the kernels have ssim0, and the kernels
        # add fp32 per-pixel SSIMs in partial sums before the double accumulation: per pixel at
        # most 1 - ssim0 plus a rounding of ~2^-24 per level of a (log-depth) shuffle tree, i.e.
        # |d mean SSIM| <= |1 - ssim0| + 16 * 2^-24; L1 is exact outside the patches.
        want_loss = (1 - lam) * l1_sum / n_full + lam * (1.0 - (ss_sum + (n_full - n_crops) * ssim0) / n_full)
        tol = lam * (abs(1.0 - ssim0) + 16 * 2.0 ** -24) + 1e-5 * abs(want_loss)
        assert abs(float(loss) - want_loss) <= tol, (H, W, float(loss), want_loss, tol)
        # L1 alone (lambda = 0) has no background term: fp32 loss to a few ulps
        l0, _ = gau_loss_with_grad(img, gt, 0.0, want_grad=False)
        assert abs(float(l0) - l1_sum / n_full) <= 1e-5 * l1_sum / n_full, (H, W)
        del img, gt, loss, grad, l0
        torch.cuda.empty_cache()
    print("peak device memory %.2f GB" % (torch.cuda.max_memory_allocated() / 2**30))


@pytest.mark.gpu
def test_gpu_gau_loss_reference_fixture():
    from easygaussiansplatting_b200.loss import gau_loss
    d = dict(np.load(G))
    for k in "ab":
        ti = torch.from_numpy(d["img_" + k]).cuda().requires_grad_()
        loss = gau_loss(ti, torch.from_numpy(d["gt_" + k]).cuda())
        loss.backward()
        assert abs(loss.item() - float(d["loss_" + k])) < 2e-6
        ref = d["grad_" + k]
        assert np.abs(ti.grad.cpu().numpy() - ref).max() / np.abs(ref).max() < 3e-4
