"""Bilateral-grid colour correction (DESIGN 3.20; Wang et al., "Bilateral Guided Radiance Field
Processing", SIGGRAPH 2024): one small learnable grid of 3 x 4 affine colour matrices per training
image, sliced on the rendered image before the loss, so that per-photo exposure, white balance and
tone changes are fitted by the grid instead of by floaters and bent SH colours.

    bil = BilateralGrid(len(train_images), device="cuda")
    grid_opt = torch.optim.Adam(bil.parameters(), lr=2e-3)   # a second optimiser, dense
    image = bil(image, i)                                    # i: the training image's index
    loss = gau_loss(image, gt) + lambda_tv * bil.tv_loss()

`grids` is [num_images, 12, L, Y, X], not [N, D] over the Gaussians: it goes in its own optimiser,
`torch.optim.Adam` or a dense `GaussianAdam`, never the selective (visibility-masked) step, and it
is untouched by density control.  The slice and its backward are CUDA kernels (csrc/bilagrid.cu);
there is no torch fallback.
"""
import torch

from . import ops

_IDENTITY = (1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0)  # A = [I | 0], row-major


class _BilagridSlice(torch.autograd.Function):
    @staticmethod
    def forward(ctx, grids, rgb, image_ids):
        out = ops.bilagrid_slice(grids.detach(), rgb.detach(), image_ids)
        ctx.save_for_backward(grids, rgb)
        ctx.image_ids = image_ids
        return out

    @staticmethod
    def backward(ctx, dloss_dout):
        grids, rgb = ctx.saved_tensors
        drgb, dgrids = ops.bilagrid_sliceB(grids.detach(), rgb.detach(), ctx.image_ids, dloss_dout)
        return (dgrids if ctx.needs_input_grad[0] else None, drgb if ctx.needs_input_grad[1] else None, None)


class _BilagridTV(torch.autograd.Function):
    @staticmethod
    def forward(ctx, grids):
        tv, grad = ops.bilagrid_tv(grids.detach(), want_grad=True)
        ctx.save_for_backward(grad)
        return tv.reshape(())

    @staticmethod
    def backward(ctx, grad_output):
        (grad,) = ctx.saved_tensors
        return grad * grad_output


def bilateral_slice(grids, rgb, image_ids):
    """Differentiable slice of rgb ([3,H,W] with one index, or [B,3,H,W] with B indices, host
    integers) through grids[M, 12, L, Y, X]; per pixel, with g = 0.299 r + 0.587 g + 0.114 b,
    A = grids[i] interpolated trilinearly at ((px + 1/2) / W (X - 1), (py + 1/2) / H (Y - 1),
    clamp(g, 0, 1) (L - 1)) and out = A[:, :3] rgb + A[:, 3].  Gradients reach grids and rgb (rgb's
    through A and through g).  Two batch items naming one grid add up into its gradient."""
    return _BilagridSlice.apply(grids, rgb, image_ids)


def total_variation(grids):
    """TV(grids) = sum over the axes a in {L, Y, X} of mean((grids shifted by one along a - grids)^2),
    each mean over every grid's differences along a; an axis of size 1 contributes 0.  gsplat's
    `total_variation_loss` also divides this sum by the number of grids, so its lambda_tv is M times
    the one that gives the same regularisation here.  Differentiable w.r.t. grids."""
    return _BilagridTV.apply(grids)


class BilateralGrid(torch.nn.Module):
    """num_images grids of grid_X x grid_Y x grid_L vertices (each 1 to 64), initialised to the
    identity.  forward(rgb, image_ids) slices a rendered image (or a batch), tv_loss() is
    `total_variation` of all grids.  The grids are saved with the module's state_dict."""

    def __init__(self, num_images, grid_X=16, grid_Y=16, grid_L=8, device="cuda"):
        super().__init__()
        ident = torch.tensor(_IDENTITY, dtype=torch.float32).view(1, 12, 1, 1, 1)
        grids = ident.repeat(int(num_images), 1, int(grid_L), int(grid_Y), int(grid_X))
        ops._bilagrid_dims(grids.shape)
        self.grids = torch.nn.Parameter(grids.to(device))

    @property
    def num_images(self):
        return self.grids.shape[0]

    def forward(self, rgb, image_ids):
        return bilateral_slice(self.grids, rgb, image_ids)

    def tv_loss(self):
        return total_variation(self.grids)
