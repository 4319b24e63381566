"""Fused training loss (SURVEY 8f row N2): a drop-in for the reference's
`gsplat.pytorch_ssim.gau_loss(image, gt_image, loss_lambda=0.2)` (pytorch_ssim.py:64-67, used at
train.py:52).  One call computes the loss and dloss/dimage on the GPU (two HBM-bound kernels,
csrc/loss.cu); autograd only scales the stored gradient by the incoming grad_output.

Swap-in for train.py:  `from easygaussiansplatting_b200.loss import gau_loss`.
"""
import torch

from . import _lib
from .ops import _chk, _L, _ptr, _same_device, _stream


def gau_loss_with_grad(image, gt_image, loss_lambda=0.2, want_grad=True):
    """-> (loss scalar tensor [1], dloss_dimage [3,H,W] or None)"""
    image = _chk(image, "image", ndim=3); gt = _chk(gt_image, "gt_image", ndim=3)
    _same_device(image, gt)
    if image.shape != gt.shape or image.shape[0] != 3:
        raise ValueError("image and gt_image must both be [3,H,W], got %s and %s" % (tuple(image.shape), tuple(gt.shape)))
    H, W = int(image.shape[1]), int(image.shape[2])
    lib = _L()
    loss = torch.empty((1,), dtype=torch.float32, device=image.device)
    grad = torch.empty_like(image) if want_grad else None
    with torch.cuda.device(image.device):
        ws_bytes = lib.gsb_gau_loss_workspace_bytes(H, W)
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=image.device)
        _lib.check(lib.gsb_gau_loss(H, W, _ptr(image), _ptr(gt), float(loss_lambda), _ptr(loss), _ptr(grad), _ptr(ws),
                                    ws_bytes, _stream()), lib)
    return loss, grad


class _GauLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, gt_image, loss_lambda):
        loss, grad = gau_loss_with_grad(image.detach(), gt_image.detach(), loss_lambda, want_grad=True)
        ctx.save_for_backward(grad)
        return loss.reshape(())

    @staticmethod
    def backward(ctx, grad_output):
        (grad,) = ctx.saved_tensors
        return grad * grad_output, None, None


def gau_loss(image, gt_image, loss_lambda=0.2):
    """Same signature and value as the reference's gau_loss; differentiable w.r.t. `image`."""
    return _GauLoss.apply(image, gt_image, loss_lambda)


def depth_to_normal(depth, cam):
    """The camera-frame normal of a depth map, for 2D Gaussian Splatting's depth-normal consistency
    term (DESIGN 3.16).  Pure torch, differentiable by autograd; no kernel.
    depth[H,W] (or [1,H,W]): camera-frame z per pixel, e.g. GSFunctionSurfelGeometry's median_depth
    or depth / alpha.  Each pixel is unprojected through the pinhole K of `cam` (fx, fy, cx, cy) to
    X(u, v) = depth (u - cx) / fx, depth (v - cy) / fy, depth); the normal is the unit cross product of
    the central differences X(u+1, v) - X(u-1, v) and X(u, v+1) - X(u, v-1), oriented to face the
    camera (n . X <= 0), which is the surfel normal plane's convention: -z for a fronto-parallel
    plane.  -> [3,H,W]; the one-pixel border is 0.
    A pixel without a surface to differentiate gets a zero normal with a zero gradient: one whose own
    depth or a neighbour's is <= 0 (median_depth is 0 where nothing contributes: a thin covered strip
    against an empty background has no vertical difference), or whose cross product is exactly 0.
    2DGS's normal term (alpha detached, as there) is then
        L_n = (1 - (normal * depth_to_normal(median_depth, cam) * alpha.detach()).sum(0)).mean()
    with normal and alpha GSFunctionSurfelGeometry's planes (its normal plane is sum w n).
    A batch (GSFunctionSurfelGeometryBatch, DESIGN 3.25): depth[C,H,W] with `cam` a list of C cameras
    -> [C,3,H,W], frame c the normal of depth[c] through cam[c]."""
    if isinstance(cam, (list, tuple)):
        if depth.dim() != 3 or depth.shape[0] != len(cam):
            raise ValueError("depth must be [C, H, W] for a list of C cameras, got %s for %d cameras"
                             % (tuple(depth.shape), len(cam)))
        return torch.stack([depth_to_normal(depth[c], cam[c]) for c in range(len(cam))])
    d = depth.reshape(depth.shape[-2], depth.shape[-1])
    H, W = d.shape
    v, u = torch.meshgrid(torch.arange(H, dtype=d.dtype, device=d.device),
                          torch.arange(W, dtype=d.dtype, device=d.device), indexing="ij")
    X = torch.stack([d * (u - float(cam.cx)) / float(cam.fx), d * (v - float(cam.cy)) / float(cam.fy), d])
    dx = X[:, 1:-1, 2:] - X[:, 1:-1, :-2]
    dy = X[:, 2:, 1:-1] - X[:, :-2, 1:-1]
    n = torch.linalg.cross(dx, dy, dim=0)
    sq = (n * n).sum(0, keepdim=True)
    valid = ((d[1:-1, 1:-1] > 0) & (d[1:-1, 2:] > 0) & (d[1:-1, :-2] > 0) & (d[2:, 1:-1] > 0) &
             (d[:-2, 1:-1] > 0))[None] & (sq > 0)
    # both branches finite, and the invalid one constant: no gradient reaches a degenerate pixel
    n = torch.where(valid, n * torch.rsqrt(torch.where(valid, sq, torch.ones_like(sq))), torch.zeros_like(n))
    n = torch.where((n * X[:, 1:-1, 1:-1]).sum(0, keepdim=True) > 0, -n, n)
    return torch.nn.functional.pad(n, (1, 1, 1, 1))
