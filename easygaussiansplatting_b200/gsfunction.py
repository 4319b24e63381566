"""Host-side mirror of the reference's autograd wrapper (gsplat/gsmodel.py:6-93).

`GSFunction.apply(pws, shs, alphas, scales, rots, us, cam)` has the reference's argument
order, return values (image, depths > 0.2 mask) and gradient slots, and drives the same
seven operators in the same order, so it is the caller contract the parity and benchmark
harnesses exercise on the GPU box (where the reference tree itself is not available).
The reference's own gsplat/gsmodel.py runs unmodified on top of `gsplatcu` as well.
"""
import math

import torch


class Camera:
    """Fields of gsplat/gausplat_dataset.py:14-27 that the rasterizer reads.  antialiased (an
    extension, read by the fused classes, GraphedFusedStep and MultiViewStep): render with the
    2D-filter opacity compensation, alpha_eff = rho * alpha (ops.preprocess).
    camera_model (an extension, read by the same classes): "pinhole" (the reference's projection),
    "ortho" (u = (fx x + cx, fy y + cy)), "fisheye" (Kannala-Brandt, COLMAP's OPENCV_FISHEYE, with
    radial_coeffs = (k1, k2, k3, k4); None = the equidistant lens) or "opencv" (radial-tangential,
    COLMAP's OPENCV / RADIAL / SIMPLE_RADIAL, with radial_coeffs = (k1, k2) and tangential_coeffs =
    (p1, p2); None = 0).  `colmap_intrinsics` maps COLMAP's camera records onto these fields.  The
    seven-operator GSFunction, GradExchange, the surfel classes, the 3D filter's camera table and
    TSDF fusion take pinhole cameras only."""

    def __init__(self, width, height, fx, fy, cx, cy, Rcw, tcw, twc=None, antialiased=False, camera_model="pinhole",
                 radial_coeffs=None, tangential_coeffs=None):
        from .ops import camera_model_args
        self.width, self.height = int(width), int(height)
        self.fx, self.fy, self.cx, self.cy = float(fx), float(fy), float(cx), float(cy)
        self.Rcw, self.tcw = Rcw, tcw
        self.twc = twc if twc is not None else -torch.linalg.inv(Rcw) @ tcw
        self.antialiased = bool(antialiased)
        self.camera_model, k = camera_model_args(camera_model, radial_coeffs, tangential_coeffs)
        nk = 2 if self.camera_model == "opencv" else 4
        self.radial_coeffs = k[:nk] if radial_coeffs is not None else None
        self.tangential_coeffs = k[2:] if tangential_coeffs is not None else None
        if self.camera_model != "pinhole" and not (self.fx > 0 and self.fy > 0):
            raise ValueError("camera_model=%r needs fx, fy > 0" % self.camera_model)


def camera_model_kwargs(cam):
    """ops.preprocess / preprocessB keywords of a camera; one without the fields (the reference's
    dataset Camera) is pinhole"""
    return dict(camera_model=getattr(cam, "camera_model", "pinhole"), radial_coeffs=getattr(cam, "radial_coeffs", None),
                tangential_coeffs=getattr(cam, "tangential_coeffs", None))


# COLMAP camera model -> (number of params, camera_model); params as in COLMAP's cameras.txt / .bin
_COLMAP_MODELS = {"SIMPLE_PINHOLE": (3, "pinhole"), "PINHOLE": (4, "pinhole"), "SIMPLE_RADIAL": (4, "opencv"),
                  "RADIAL": (5, "opencv"), "OPENCV": (8, "opencv"), "OPENCV_FISHEYE": (8, "fisheye")}


def colmap_intrinsics(model_name, params, width, height, image_width=None, image_height=None):
    """The `Camera` fields of a COLMAP camera record -> dict(fx, fy, cx, cy, camera_model, radial_coeffs,
    tangential_coeffs), for images resized from (width, height) to (image_width, image_height) (default:
    not resized).  Focal lengths and the principal point scale with the image; distortion coefficients
    are in normalised coordinates and do not.
      SIMPLE_PINHOLE f, cx, cy            -> pinhole
      PINHOLE        fx, fy, cx, cy       -> pinhole
      SIMPLE_RADIAL  f, cx, cy, k         -> opencv, radial (k, 0)
      RADIAL         f, cx, cy, k1, k2    -> opencv, radial (k1, k2)
      OPENCV         fx, fy, cx, cy, k1, k2, p1, p2 -> opencv
      OPENCV_FISHEYE fx, fy, cx, cy, k1, k2, k3, k4 -> fisheye
    Any other model, or a wrong number of params, is a ValueError.  Reads no files."""
    if model_name not in _COLMAP_MODELS:
        raise ValueError("COLMAP camera model %r is not supported (one of %s)" % (model_name, tuple(_COLMAP_MODELS)))
    n, camera_model = _COLMAP_MODELS[model_name]
    p = [float(v) for v in params]
    if len(p) != n:
        raise ValueError("COLMAP camera model %s takes %d params, got %d" % (model_name, n, len(p)))
    if model_name in ("SIMPLE_PINHOLE", "SIMPLE_RADIAL", "RADIAL"):
        fx = fy = p[0]
        cx, cy, rest = p[1], p[2], p[3:]
    else:
        fx, fy, cx, cy, rest = p[0], p[1], p[2], p[3], p[4:]
    sx = 1.0 if image_width is None else float(image_width) / float(width)
    sy = 1.0 if image_height is None else float(image_height) / float(height)
    radial = tangential = None
    if model_name == "SIMPLE_RADIAL":
        radial = (rest[0], 0.0)
    elif model_name == "RADIAL":
        radial = tuple(rest)
    elif model_name == "OPENCV":
        radial, tangential = tuple(rest[:2]), tuple(rest[2:])
    elif model_name == "OPENCV_FISHEYE":
        radial = tuple(rest)
    return dict(fx=fx * sx, fy=fy * sy, cx=cx * sx, cy=cy * sy, camera_model=camera_model, radial_coeffs=radial,
                tangential_coeffs=tangential)


def _pinhole_only(cam, what):
    if getattr(cam, "camera_model", "pinhole") != "pinhole":
        raise ValueError("%s takes pinhole cameras only, got camera_model=%r" % (what, cam.camera_model))


def _intrinsics_rows(intrinsics, shape):
    """the host values of the pose classes' `intrinsics` tensor ([8] or [C, 8], fx, fy, cx, cy, k[4]): a
    CUDA tensor costs one small device-to-host copy and a wait, a CPU tensor neither"""
    if not isinstance(intrinsics, torch.Tensor) or not intrinsics.dtype.is_floating_point or \
            tuple(intrinsics.shape) != shape:
        raise ValueError("intrinsics must be a float tensor of shape %s, got %s"
                         % (list(shape), tuple(getattr(intrinsics, "shape", ()))))
    rows = intrinsics.detach().to(device="cpu", dtype=torch.float32).reshape(-1, 8).tolist()
    if not all(math.isfinite(v) for r in rows for v in r):
        raise ValueError("intrinsics must be finite")
    return rows


def _with_intrinsics(cam, row):
    """a Camera with cam's size, pose, model and antialiasing and the intrinsics row (fx, fy, cx, cy,
    k[4]): opencv's k = (k1, k2, p1, p2), fisheye's k1..k4, 0 for pinhole and ortho"""
    model = getattr(cam, "camera_model", "pinhole")
    fx, fy, cx, cy, k = row[0], row[1], row[2], row[3], tuple(row[4:])
    radial = tangential = None
    if model in ("pinhole", "ortho"):
        if any(k):
            raise ValueError("intrinsics: k must be 0 for camera_model=%r, got %s" % (model, k))
    elif model == "opencv":
        radial, tangential = k[:2], k[2:]
    else:
        radial = k
    out = Camera(cam.width, cam.height, fx, fy, cx, cy, cam.Rcw, cam.tcw, cam.twc,
                 antialiased=getattr(cam, "antialiased", False), camera_model=model, radial_coeffs=radial,
                 tangential_coeffs=tangential)
    for name, value in vars(cam).items():  # the caller's other fields (grad_exchange, ...) come along
        if name not in vars(out):
            setattr(out, name, value)
    return out


def build_gsfunction(gsc):
    """Binds the wrapper to an operator module exposing the seven `gsplatcu` functions: ours
    (easygaussiansplatting_b200.ops) or, in benchmarks/compare_ref_gpu.py, the reference's own
    compiled extension -- the same harness drives both (SURVEY 8d "apples-to-apples")."""

    class GSFunction(torch.autograd.Function):
        @staticmethod
        def forward(ctx, pws, shs, alphas, scales, rots, us, cam):
            return _forward(gsc, ctx, pws, shs, alphas, scales, rots, us, cam)

        @staticmethod
        def backward(ctx, dloss_dgammas, _):
            return _backward(gsc, ctx, dloss_dgammas)

    return GSFunction


class _Impl:
    @staticmethod
    def forward(gsc, ctx, pws, shs, alphas, scales, rots, us, cam):
        if getattr(cam, "antialiased", False):
            raise ValueError("GSFunction (the seven-operator surface) has no antialiased mode: use GSFunctionFused")
        _pinhole_only(cam, "GSFunction (the seven-operator surface; use GSFunctionFused)")
        us, pcs, depths, du_dpcs = gsc.project(pws, cam.Rcw, cam.tcw, cam.fx, cam.fy, cam.cx, cam.cy, True)
        cov3ds, dcov3d_drots, dcov3d_dscales = gsc.computeCov3D(rots, scales, depths, True)
        cov2ds, dcov2d_dcov3ds, dcov2d_dpcs = gsc.computeCov2D(
            cov3ds, pcs, cam.Rcw, depths, cam.fx, cam.fy, cam.width, cam.height, True)
        colors, dcolor_dshs, dcolor_dpws = gsc.sh2Color(shs, pws, cam.twc, True)
        cinv2ds, areas, dcinv2d_dcov2ds = gsc.inverseCov2D(cov2ds, depths, True)
        image, contrib, final_tau, patch_range_per_tile, gsid_per_patch = gsc.splat(
            cam.height, cam.width, us, cinv2ds, alphas, depths, colors, areas)
        ctx.cam = cam
        ctx.alpha_shape = alphas.shape
        ctx.save_for_backward(us, cinv2ds, alphas, depths, colors, contrib, final_tau,
                              patch_range_per_tile, gsid_per_patch, dcinv2d_dcov2ds, dcov2d_dcov3ds,
                              dcov3d_drots, dcov3d_dscales, dcolor_dshs, du_dpcs, dcov2d_dpcs,
                              dcolor_dpws)
        return image, depths > 0.2

    @staticmethod
    def backward(gsc, ctx, dloss_dgammas):
        cam = ctx.cam
        (us, cinv2ds, alphas, depths, colors, contrib, final_tau, patch_range_per_tile,
         gsid_per_patch, dcinv2d_dcov2ds, dcov2d_dcov3ds, dcov3d_drots, dcov3d_dscales, dcolor_dshs,
         du_dpcs, dcov2d_dpcs, dcolor_dpws) = ctx.saved_tensors
        dloss_dus, dloss_dcinv2ds, dloss_dalphas, dloss_dcolors = gsc.splatB(
            cam.height, cam.width, us, cinv2ds, alphas, depths, colors, contrib, final_tau,
            patch_range_per_tile, gsid_per_patch, dloss_dgammas)
        # docs/backward.md eq. (3)-(7): chain through the saved per-Gaussian Jacobians
        R = cam.Rcw
        dloss_dcov2ds = dloss_dcinv2ds @ dcinv2d_dcov2ds
        dloss_dcov3ds = dloss_dcov2ds @ dcov2d_dcov3ds
        dloss_drots = dloss_dcov3ds @ dcov3d_drots
        dloss_dscales = dloss_dcov3ds @ dcov3d_dscales
        n = dloss_dcolors.shape[0]
        dloss_dshs = (dloss_dcolors.transpose(1, 2) @ dcolor_dshs).transpose(1, 2).reshape(n, -1)
        dloss_dpws = (dloss_dus @ du_dpcs + dloss_dcov2ds @ dcov2d_dpcs) @ R + dloss_dcolors @ dcolor_dpws
        return (dloss_dpws.squeeze(1), dloss_dshs, dloss_dalphas.reshape(ctx.alpha_shape), dloss_dscales.squeeze(1),
                dloss_drots.squeeze(1), dloss_dus.squeeze(1), None)


_forward, _backward = _Impl.forward, _Impl.backward


def __getattr__(name):
    if name == "GSFunction":  # bound lazily so importing this module does not load the library
        from . import ops
        cls = build_gsfunction(ops)
        globals()["GSFunction"] = cls
        return cls
    raise AttributeError(name)


class GSFunctionFused(torch.autograd.Function):
    """Same call signature, outputs and gradient slots as GSFunction, but the per-Gaussian
    stages run as one fused forward kernel and one fused backward kernel (ops.preprocess /
    ops.preprocessB) instead of five Jacobian-materialising ops + the torch.bmm chain.
    Swap-in: `from easygaussiansplatting_b200.gsfunction import GSFunctionFused as GSFunction`
    in gsplat/gsmodel.py.
    All four fused classes take an optional trailing `filter3d[N]` (ops.filter3d; after `cam`):
    the Mip-Splatting 3D filter, a constant that gets no gradient.  The frame is then rendered from
    s', alpha' (ops.filter3d_apply) and the scale and opacity gradients are taken back through it.
    They also take an optional `us_abs[N,2]` after filter3d (absolute-gradient densification, AbsGS):
    a dummy input, normally zeros with requires_grad=True, whose gradient is the per-pixel absolute
    sum of dL/du (ops.splatB(..., absgrad=True)), as `us` is the dummy whose gradient is dL/du.
    `DensityController.update_density_info(us_abs.grad, mask)` then densifies on it.  The
    rasterizer's _abs kernel runs only when us_abs requires a gradient; every other gradient is the
    one the call without us_abs returns.  Single view: refused with cam.grad_exchange."""

    @staticmethod
    def forward(ctx, pws, shs, alphas, scales, rots, us, cam, filter3d=None, us_abs=None):
        return _fused_forward(ctx, False, pws, shs, alphas, scales, rots, us, cam, filter3d=filter3d, us_abs=us_abs)

    @staticmethod
    def backward(ctx, dloss_dgammas, _):
        return _fused_backward(ctx, False, False, dloss_dgammas)


class GSFunctionFusedRGBD(torch.autograd.Function):
    """GSFunctionFused with depth and opacity: the same arguments and gradient slots, outputs
    (image[3,H,W], depth[H,W], alpha[H,W], depths > 0.2) with
        depth[p] = sum_i w_i(p) z_i,   alpha[p] = sum_i w_i(p)
    (w = tau alpha', the image's compositing weights; z = camera-frame depth).  depth is not
    normalised: depth / alpha is the expected depth.  Gradients of all three images flow to pws,
    shs, alphas, scales, rots and us; the depth term reaches pws through z = (Rcw pw + tcw)[2].
    us_abs (after filter3d) as for GSFunctionFused: its gradient sums the per-pixel terms of all
    three planes."""

    @staticmethod
    def forward(ctx, pws, shs, alphas, scales, rots, us, cam, filter3d=None, us_abs=None):
        return _fused_forward(ctx, True, pws, shs, alphas, scales, rots, us, cam, filter3d=filter3d, us_abs=us_abs)

    @staticmethod
    def backward(ctx, dloss_dgammas, dloss_ddepth, dloss_dalpha, _):
        return _fused_backward(ctx, True, False, dloss_dgammas, dloss_ddepth, dloss_dalpha)


def _fused_forward(ctx, rgbd, pws, shs, alphas, scales, rots, us, cam, pose=None, filter3d=None, features=None,
                   us_abs=None, intrinsics=None):
    """The forward of the fused classes: the colour or (rgbd) RGB-D frame.  pose: None (the
    camera is cam.Rcw, cam.tcw, cam.twc) or the tensors (Rcw, tcw, twc), then saved for the backward.
    cam.antialiased (absent: False): the rasterizers composite alpha_eff = rho * alpha.
    filter3d: None, or the Mip-Splatting 3D filter[N] (ops.filter3d, a constant): the frame is
    rendered from s' = sqrt(s^2 + f^2) and alpha' = alpha prod s / s' (ops.filter3d_apply).
    features: None, or [N, D]: the feature map [D, H, W] follows the image (ops.splat_features,
    from the same records) and features is saved last.
    us_abs: None, or the [N,2] dummy input whose gradient is the absolute-gradient statistic; its
    gradient slot (after cam and filter3d) is kept in ctx.abs_slot.
    intrinsics (pose classes): None, or the [8] tensor whose values replace cam's intrinsics and lens
    (DESIGN 3.23); its gradient slot (after us_abs) is kept in ctx.intr_slot."""
    from . import ops
    ctx.abs_slot = ctx.intr_slot = None
    if intrinsics is not None:
        cam = _with_intrinsics(cam, _intrinsics_rows(intrinsics, (8,))[0])
        ctx.intr_slot = 12
        ctx.intr_like = (intrinsics.device, intrinsics.dtype, intrinsics.shape)
    if getattr(cam, "grad_exchange", None) is not None:
        _pinhole_only(cam, "the gradient exchange (cam.grad_exchange)")
    if us_abs is not None:
        if getattr(cam, "grad_exchange", None) is not None:
            raise ValueError("us_abs is single-view: cam.grad_exchange must not be set")
        if not isinstance(us_abs, torch.Tensor) or tuple(us_abs.shape) != (pws.shape[0], 2):
            raise ValueError("us_abs must be a [N, 2] tensor (N = %d), got %s"
                             % (pws.shape[0], tuple(getattr(us_abs, "shape", ()))))
        if us_abs.device != pws.device:
            raise ValueError("us_abs must be on the device of pws (%s), got %s" % (pws.device, us_abs.device))
        ctx.abs_slot = 6 + (3 if pose is not None else 0) + 2
    ctx.filtered = filter3d is not None
    raw = ()
    if ctx.filtered:
        filter3d = filter3d.detach()
        raw = (scales, alphas, filter3d)
        scales, alphas = ops.filter3d_apply(scales, alphas, filter3d)
    aa = bool(getattr(cam, "antialiased", False))
    if pose is None:
        Rcw, tcw, twc = cam.Rcw, cam.tcw, cam.twc
        if aa and not rgbd and getattr(cam, "grad_exchange", None) is not None:
            raise ValueError("the gradient exchange has no antialiased form: cam.grad_exchange must not be set")
    else:
        if getattr(cam, "grad_exchange", None) is not None:
            raise ValueError("camera gradients are single-view: cam.grad_exchange must not be set")
        Rcw, tcw, twc = (x.detach() for x in pose)
    # the per-Gaussian records of the rasterizers come straight out of the fused forward (with z in
    # their depth word, as the RGB-D rasterizer needs)
    pre = ops.preprocess(pws, rots, scales, shs, Rcw, tcw, twc, cam.fx, cam.fy, cam.cx, cam.cy, cam.width,
                         cam.height, alphas=alphas, antialiased=aa, **camera_model_kwargs(cam))
    us, cinv2ds, colors, depths, areas, records = pre[:6]
    drawn = pre[6] if aa else alphas  # the opacities the rasterizers composite
    splat = ops.splat_rgbd if rgbd else ops.splat
    out = splat(cam.height, cam.width, us, cinv2ds, drawn, depths, colors, areas, records=records, capacity=True)
    ctx.cam = cam
    ctx.aa = aa
    ctx.alpha_shape = alphas.shape
    saved = (pws, shs, alphas, drawn, scales, rots, us, cinv2ds, depths, colors, *out[1:5])
    if pose is not None:
        ctx.cam_shapes = (Rcw.shape, tcw.shape, twc.shape)
        saved += (Rcw, tcw, twc)
    feat = ()
    if features is not None:
        feat = (features,)
        fmap = ops.splat_features(cam.height, cam.width, features, out[1], out[3], out[4], records=records)
    ctx.save_for_backward(*(saved + raw + feat))  # (with the filter, scales and alphas above are s', alpha')
    mask = depths > 0.2
    if features is not None:
        return out[0], fmap, mask
    return (out[0], out[5], out[6], mask) if rgbd else (out[0], mask)


def _fused_backward(ctx, rgbd, pose, dloss_dgammas, dloss_ddepth=None, dloss_dalpha=None, featured=False,
                    dloss_dfeatures_map=None):
    """The backward of the fused classes -> the gradients of the map inputs (pws, shs, alphas,
    scales, rots, us), with pose those of Rcw, tcw, twc, with features (featured) that of features,
    and None for cam (and filter3d).  What runs follows ctx.needs_input_grad: the pose alone takes
    the pose-only kernel (a frozen map: tracking)."""
    from . import ops
    cam = ctx.cam
    (pws, shs, alphas, drawn, scales, rots, us, cinv2ds, depths, colors, contrib, final_tau, patch_range_per_tile,
     gsid_per_patch, *rest) = ctx.saved_tensors
    if featured:
        feat = (rest.pop(), dloss_dfeatures_map)
    Rcw, tcw, twc = rest[:3] if pose else (cam.Rcw, cam.tcw, cam.twc)
    raw = rest[3:] if pose else rest  # (scales, alphas, filter3d) of a filtered frame
    need_abs = ctx.abs_slot is not None and ctx.needs_input_grad[ctx.abs_slot]
    need_intr = ctx.intr_slot is not None and ctx.needs_input_grad[ctx.intr_slot]
    grads = _fused_backward_core(ctx, rgbd, pose, ops, cam, pws, shs, alphas, drawn, scales, rots, us, cinv2ds,
                                 depths, colors, contrib, final_tau, patch_range_per_tile, gsid_per_patch, Rcw, tcw,
                                 twc, dloss_dgammas, dloss_ddepth, dloss_dalpha, feat if featured else None,
                                 absgrad=need_abs, intr=need_intr)
    if need_intr:
        grads, dintr = grads[:-1], grads[-1]
    if need_abs:
        grads, dabs = grads[:-1], grads[-1]
    if featured:  # dL/dfeatures goes right after the map inputs (the pose classes take no features)
        grads, dfeat = grads[:-1], grads[-1]
    if ctx.filtered and grads[3] is not None:
        # the gradients are those of s', alpha' (summed over the ranks with the exchange: the filter's
        # backward is linear with per-Gaussian coefficients, so it applies after the sum as well)
        dscales, dalphas = ops.filter3d_backward(*raw, grads[3], grads[2], inplace=True)
        grads = grads[:2] + (dalphas, dscales) + grads[4:]
    if featured:
        grads = grads + (dfeat,)
    if need_abs:  # cam and filter3d get None, us_abs the statistic
        grads = grads + (None,) * (ctx.abs_slot - len(grads)) + (dabs,)
    if need_intr:
        dev, dtype, shape = ctx.intr_like
        grads = grads + (None,) * (ctx.intr_slot - len(grads)) + (dintr.to(device=dev, dtype=dtype).reshape(shape),)
    # one gradient per input apply received (cam, and filter3d when passed -- also as None -- get None)
    return grads + (None,) * (len(ctx.needs_input_grad) - len(grads))


def _fused_backward_core(ctx, rgbd, pose, ops, cam, pws, shs, alphas, drawn, scales, rots, us, cinv2ds, depths,
                         colors, contrib, final_tau, patch_range_per_tile, gsid_per_patch, Rcw, tcw, twc,
                         dloss_dgammas, dloss_ddepth, dloss_dalpha, feat=None, absgrad=False, intr=False):
    """the gradients of the inputs the frame was rendered from, up to and including the pose's;
    feat: None, or (features, dL/dfeature map or None) -> dL/dfeatures (None when no map gradient
    came) appended; absgrad: the rasterizer's _abs kernel runs and its dloss_dus_abs[N,2] is
    appended; intr (pose): dL/dintrinsics[8] is appended last"""
    need_map = any(ctx.needs_input_grad[:6])
    need_pose = pose and any(ctx.needs_input_grad[6:9])
    need_cam = need_pose or intr
    # the rasterizer backward leaves its raw moment rows; the fused per-Gaussian backward converts
    # them in registers (no finalize pass, no 32 B/Gaussian round trip).  (autograd hands zeros for
    # an RGB-D output the loss does not use: all three planes are given)  With antialiasing the
    # rasterizer replays alpha_eff (`drawn`), and the per-Gaussian backward takes the raw alphas.
    ddepths = dabs = None
    if rgbd:
        rb = ops.splatB_rgbd(cam.height, cam.width, us, cinv2ds, drawn, depths, colors, contrib, final_tau,
                             patch_range_per_tile, gsid_per_patch, dloss_dgammas, dloss_ddepth, dloss_dalpha,
                             moments_only=True, absgrad=absgrad)
        moments, ddepths = rb[:2]
        if absgrad:
            dabs = rb[2]
    elif dloss_dgammas is None:  # (the feature class: no image gradient, no colour replay)
        moments = torch.zeros((pws.shape[0], 9), dtype=torch.float32, device=pws.device)
    elif absgrad:
        moments, dabs = ops.splatB(cam.height, cam.width, us, cinv2ds, drawn, depths, colors, contrib, final_tau,
                                   patch_range_per_tile, gsid_per_patch, dloss_dgammas, moments_only=True,
                                   absgrad=True)
    else:
        moments = ops.splatB(cam.height, cam.width, us, cinv2ds, drawn, depths, colors, contrib, final_tau,
                             patch_range_per_tile, gsid_per_patch, dloss_dgammas, moments_only=True)
    dfeat = None
    if feat is not None and feat[1] is not None:
        # the feature map's terms are added to moment rows 0-5: the conversion below sums both losses
        moments, dfeat = ops.splatB_features(cam.height, cam.width, feat[0], contrib, final_tau, patch_range_per_tile,
                                             gsid_per_patch, feat[1], moments=moments, us=us, cinv2ds=cinv2ds,
                                             alphas=drawn, colors=colors)
    ex = None if rgbd or pose else getattr(cam, "grad_exchange", None)
    if ex is not None:
        # multi-view data parallel (parallel.GradExchange): the per-Gaussian backward pushes
        # its tiles into peer memory and the gradients come back already summed over ranks
        # (dloss_dus stays this view's own: it only feeds the densification statistics)
        g = ex.backward(pws, rots, scales, shs, cam, moments=moments, cinv2ds=cinv2ds)
        # the result region is overwritten by the next step's broadcast: hand autograd its own
        # copies (AccumulateGrad may keep a returned tensor, and so may hooks / retain_grad)
        return (g["dpws"].clone(), g["dshs"].clone(), g["dalphas"].clone().reshape(ctx.alpha_shape),
                g["dscales"].clone(), g["drots"].clone(), g["dus"])
    out = ops.preprocessB(pws, rots, scales, shs, Rcw, tcw, twc, cam.fx, cam.fy, cam.cx, cam.cy, cam.width,
                          cam.height, None, None, None, moments=moments, cinv2ds=cinv2ds, dloss_ddepths=ddepths,
                          camera_grad=need_cam, pose_only=need_cam and not need_map, antialiased=ctx.aa,
                          alphas=alphas if ctx.aa else None, intrinsics_grad=intr, **camera_model_kwargs(cam))
    if need_map:
        dpws, dshs, dscales, drots, dloss_dus, dloss_dalphas = out[:6]
        grads = (dpws, dshs, dloss_dalphas.reshape(ctx.alpha_shape), dscales, drots, dloss_dus)
    else:
        grads = (None,) * 6
    if need_pose:
        grads += tuple(d.reshape(s) for d, s in zip(out[6], ctx.cam_shapes))
    elif pose:
        grads += (None, None, None)
    if absgrad:
        grads += (dabs,)
    if intr:
        grads += (out[-1],)
    return grads + (dfeat,) if feat is not None else grads


class GSFunctionFusedBatch(torch.autograd.Function):
    """GSFunctionFused for C cameras in one call (DESIGN 3.21): `apply(pws, shs, alphas, scales, rots,
    us, cams, filter3d=None)` -> (image[C,3,H,W], mask[C,N]) with image[c] and mask[c] those of
    camera cams[c].  The cameras share width, height, antialiased and camera_model (else ValueError);
    each has its own pose, intrinsics and lens coefficients.  us is the [C,N,2] dummy whose gradient
    is each camera's dL/du, so `DensityController.update_density_info(us.grad[c], mask[c])` works per
    camera.  The map gradients are the sums over the cameras, taken in one per-Gaussian pass.
    filter3d: as for GSFunctionFused, applied once per call.  Poses with gradients: GSFunctionFusedBatchPose
    (DESIGN 3.22).  No features, AbsGS or gradient exchange in batch form."""

    @staticmethod
    def forward(ctx, pws, shs, alphas, scales, rots, us, cams, filter3d=None):
        return _batch_forward(ctx, False, pws, shs, alphas, scales, rots, us, cams, filter3d)

    @staticmethod
    def backward(ctx, dloss_dimage, _):
        return _batch_backward(ctx, dloss_dimage)


class GSFunctionFusedBatchRGBD(torch.autograd.Function):
    """GSFunctionFusedBatch with GSFunctionFusedRGBD's planes: -> (image[C,3,H,W], depth[C,H,W],
    alpha[C,H,W], mask[C,N])"""

    @staticmethod
    def forward(ctx, pws, shs, alphas, scales, rots, us, cams, filter3d=None):
        return _batch_forward(ctx, True, pws, shs, alphas, scales, rots, us, cams, filter3d)

    @staticmethod
    def backward(ctx, dloss_dimage, dloss_ddepth, dloss_dalpha, _):
        return _batch_backward(ctx, dloss_dimage, dloss_ddepth, dloss_dalpha)


class GSFunctionFusedBatchPose(torch.autograd.Function):
    """GSFunctionFusedBatch with differentiable camera poses (DESIGN 3.22):
    `apply(pws, shs, alphas, scales, rots, us, Rcws, tcws, twcs, cams, filter3d=None)` -> (image[C,3,H,W],
    mask[C,N]).  Rcws[C,3,3], tcws[C,3], twcs[C,3] replace the cameras' own poses (cams supply size,
    intrinsics, lens, camera model and antialiasing) and get dL/dRcw, dL/dtcw, dL/dtwc per camera as
    independent inputs, as GSFunctionFusedPose's do: a caller who builds twcs from the other two has
    autograd chain it.  What runs follows ctx.needs_input_grad: only the poses -> the pose-only pass (a
    frozen map: tracking several frames, or the poses' step of windowed bundle adjustment); no pose ->
    exactly GSFunctionFusedBatch's backward; both -> the pose pass, then that backward.  filter3d as for
    GSFunctionFusedBatch.
    intrinsics (after filter3d; DESIGN 3.23): None, or a float tensor [C, 8], row c as
    GSFunctionFusedPose's intrinsics for cams[c], with the same host-copy trade-off and the gradient
    per camera.  One physical camera shared by every view: pass intrinsics[None].expand(C, 8) and
    autograd sums the rows."""

    @staticmethod
    def forward(ctx, pws, shs, alphas, scales, rots, us, Rcws, tcws, twcs, cams, filter3d=None, intrinsics=None):
        return _batch_forward(ctx, False, pws, shs, alphas, scales, rots, us, cams, filter3d, (Rcws, tcws, twcs),
                              intrinsics)

    @staticmethod
    def backward(ctx, dloss_dimage, _):
        return _batch_backward(ctx, dloss_dimage)


class GSFunctionFusedBatchRGBDPose(torch.autograd.Function):
    """GSFunctionFusedBatchRGBD with differentiable camera poses, as GSFunctionFusedBatchPose:
    `apply(pws, shs, alphas, scales, rots, us, Rcws, tcws, twcs, cams, filter3d=None)` -> (image[C,3,H,W],
    depth[C,H,W], alpha[C,H,W], mask[C,N]).  The depth planes' gradients reach the poses through
    z = (Rcw pw + tcw)[2].  intrinsics (after filter3d) as for GSFunctionFusedBatchPose."""

    @staticmethod
    def forward(ctx, pws, shs, alphas, scales, rots, us, Rcws, tcws, twcs, cams, filter3d=None, intrinsics=None):
        return _batch_forward(ctx, True, pws, shs, alphas, scales, rots, us, cams, filter3d, (Rcws, tcws, twcs),
                              intrinsics)

    @staticmethod
    def backward(ctx, dloss_dimage, dloss_ddepth, dloss_dalpha, _):
        return _batch_backward(ctx, dloss_dimage, dloss_ddepth, dloss_dalpha)


def _batch_poses(pose, C, dev):
    """(Rcws, tcws, twcs) -> the [C, 15] pose rows the batch kernels read (a detached copy)"""
    shapes = ((C, 3, 3), (C, 3), (C, 3))
    for name, x, s in zip(("Rcws", "tcws", "twcs"), pose, shapes):
        if not isinstance(x, torch.Tensor) or x.numel() != s[0] * (9 if len(s) == 3 else 3) or x.shape[0] != C:
            raise ValueError("%s must be a %s tensor, got %s" % (name, list(s), tuple(getattr(x, "shape", ()))))
        if x.device != dev:
            raise ValueError("%s must be on the device of pws (%s), got %s" % (name, dev, x.device))
    return torch.cat([x.detach().reshape(C, -1).to(torch.float32) for x in pose], 1).contiguous()


def _batch_forward(ctx, rgbd, pws, shs, alphas, scales, rots, us, cams, filter3d, pose=None, intrinsics=None):
    """the forward of the batch classes; pose: None (the cameras' own poses) or (Rcws, tcws, twcs);
    intrinsics: None or the [C, 8] tensor whose rows replace the cameras' intrinsics (gradient slot 11)"""
    from . import ops
    ctx.pose = pose is not None
    ctx.intr_slot = None
    if intrinsics is not None:
        cams = list(cams)
        cams = [_with_intrinsics(c, r) for c, r in zip(cams, _intrinsics_rows(intrinsics, (len(cams), 8)))]
        ctx.intr_slot = 11
        ctx.intr_like = (intrinsics.device, intrinsics.dtype, intrinsics.shape)
    if ctx.pose:
        bc = ops.BatchCameras(cams, pws.device, poses=_batch_poses(pose, len(cams), pws.device))
        ctx.cam_shapes = tuple(x.shape for x in pose)
    else:
        bc = ops.BatchCameras(cams, pws.device)
    N = pws.shape[0]
    if not isinstance(us, torch.Tensor) or tuple(us.shape) != (bc.C, N, 2):
        raise ValueError("us must be a [C, N, 2] tensor (C = %d, N = %d), got %s"
                         % (bc.C, N, tuple(getattr(us, "shape", ()))))
    ctx.filtered = filter3d is not None
    raw = ()
    if ctx.filtered:
        filter3d = filter3d.detach()
        raw = (scales, alphas, filter3d)
        scales, alphas = ops.filter3d_apply(scales, alphas, filter3d)
    pre = ops.preprocess_batch(pws, rots, scales, shs, bc, alphas)
    us_, cinv2ds, colors, depths, areas, records = pre[:6]
    drawn = pre[6] if bc.antialiased else alphas  # (with the records the frame reads no alphas)
    out = ops.splat_batch(bc.height, bc.width, us_, cinv2ds, drawn, depths, colors, areas, records=records,
                          capacity=True, rgbd=rgbd)
    ctx.bc = bc
    ctx.rgbd = rgbd
    ctx.alpha_shape = alphas.shape
    ctx.save_for_backward(pws, shs, alphas, drawn, scales, rots, us_, cinv2ds, depths, colors, records, *out[1:5],
                          *raw)
    mask = depths > 0.2
    return (out[0], out[5], out[6], mask) if rgbd else (out[0], mask)


def _batch_backward(ctx, dloss_dimage, dloss_ddepth=None, dloss_dalpha=None):
    from . import ops
    bc = ctx.bc
    (pws, shs, alphas, drawn, scales, rots, us, cinv2ds, depths, colors, records, contrib, final_tau, ranges, gsid,
     *raw) = ctx.saved_tensors
    rb = ops.splatB_batch(bc.height, bc.width, us, cinv2ds, drawn, depths, colors, contrib, final_tau, ranges, gsid,
                          dloss_dimage, dloss_ddepth if ctx.rgbd else None, dloss_dalpha, records=records)
    moments, ddepths = rb if ctx.rgbd else (rb, None)
    need_map = any(ctx.needs_input_grad[:6])
    need_pose = ctx.pose and any(ctx.needs_input_grad[6:9])
    need_intr = ctx.intr_slot is not None and ctx.needs_input_grad[ctx.intr_slot]
    need_cam = need_pose or need_intr
    out = ops.preprocessB_batch(pws, rots, scales, shs, bc, moments, cinv2ds, dloss_ddepths=ddepths,
                                alphas=alphas if bc.antialiased else None, camera_grad=need_cam,
                                pose_only=need_cam and not need_map, intrinsics_grad=need_intr)
    if need_map:
        dpws, dshs, dscales, drots, dus, dalphas = out[:6]
        if ctx.filtered:  # the gradients are those of s', alpha'; the filter's backward runs once, after the batch sum
            dscales, dalphas = ops.filter3d_backward(*raw, dscales, dalphas, inplace=True)
        grads = (dpws, dshs, dalphas.reshape(ctx.alpha_shape), dscales, drots, dus)
    else:
        grads = (None,) * 6
    if need_pose:
        grads += tuple(d.reshape(s) for d, s in zip(out[6], ctx.cam_shapes))
    elif ctx.pose:
        grads += (None,) * 3
    if need_intr:
        dev, dtype, shape = ctx.intr_like
        grads += (None,) * (ctx.intr_slot - len(grads)) + (out[-1].to(device=dev, dtype=dtype).reshape(shape),)
    return grads + (None,) * (len(ctx.needs_input_grad) - len(grads))


class GSFunctionFusedFeatures(torch.autograd.Function):
    """GSFunctionFused with per-Gaussian features: `apply(pws, shs, alphas, scales, rots, us, features, cam,
    filter3d=None)` -> (image[3,H,W], feature_map[D,H,W], depths > 0.2) with
        feature_map[c, p] = sum_i w_i(p) features[i, c]
    (w = tau alpha', the image's compositing weights; any width D >= 1; not view-dependent, no
    offset).  Semantic or instance labels, distilled 2D features, normals, uncertainty.  Gradients
    of both maps reach features and, through the rasterizers' moment rows, pws, alphas, scales,
    rots and us (which feeds DensityController.update_density_info as for colour).  Composes with
    Camera(..., antialiased=True) and filter3d.  A map the loss does not use costs nothing in the
    backward: without an image gradient the colour replay is skipped, without a feature-map
    gradient the feature replay.  Single view: cam.grad_exchange is refused."""

    @staticmethod
    def forward(ctx, pws, shs, alphas, scales, rots, us, features, cam, filter3d=None):
        if getattr(cam, "grad_exchange", None) is not None:
            raise ValueError("GSFunctionFusedFeatures is single-view: cam.grad_exchange must not be set")
        ctx.set_materialize_grads(False)
        return _fused_forward(ctx, False, pws, shs, alphas, scales, rots, us, cam, filter3d=filter3d,
                              features=features)

    @staticmethod
    def backward(ctx, dloss_dgammas, dloss_dfeature_map, _):
        return _fused_backward(ctx, False, False, dloss_dgammas, featured=True, dloss_dfeatures_map=dloss_dfeature_map)


class GSFunctionFusedPose(torch.autograd.Function):
    """GSFunctionFused with a differentiable camera pose:
    `apply(pws, shs, alphas, scales, rots, us, Rcw, tcw, twc, cam)` -> (image, depths > 0.2).
    The camera tensors replace cam.Rcw, cam.tcw, cam.twc (cam supplies the size and intrinsics)
    and get dL/dRcw, dL/dtcw, dL/dtwc as independent inputs: a caller that builds twc from Rcw
    and tcw with torch ops has autograd chain it.  What runs follows ctx.needs_input_grad:
    only the camera -> the pose-only kernel (a frozen map: tracking); no camera -> exactly
    GSFunctionFused's backward.  Single view only.  us_abs (after filter3d) as for GSFunctionFused, also
    with the pose-only backward.
    intrinsics (after us_abs; DESIGN 3.23): None, or a float tensor [8] = (fx, fy, cx, cy, k[4]) (k:
    opencv's k1, k2, p1, p2, fisheye's k1..k4, 0 for pinhole and ortho) whose values replace cam's
    intrinsics and lens for the render and the backward (cam still supplies size, model and
    antialiasing); it gets dL/dintrinsics when it requires a gradient.  The host needs its values: a
    CUDA tensor costs a 32-byte device-to-host copy and a wait per forward, a CPU tensor neither; the
    gradient comes back on the tensor's device.  Asking for the intrinsics alone runs the camera pass
    alone (a frozen map, a fixed pose).  Tied parameters (a SIMPLE_* model's single f) are the caller's
    autograd graph: build the tensor from them with torch ops."""

    @staticmethod
    def forward(ctx, pws, shs, alphas, scales, rots, us, Rcw, tcw, twc, cam, filter3d=None, us_abs=None,
                intrinsics=None):
        return _fused_forward(ctx, False, pws, shs, alphas, scales, rots, us, cam, (Rcw, tcw, twc), filter3d,
                              us_abs=us_abs, intrinsics=intrinsics)

    @staticmethod
    def backward(ctx, dloss_dgammas, _):
        return _fused_backward(ctx, False, True, dloss_dgammas)


class GSFunctionFusedRGBDPose(torch.autograd.Function):
    """GSFunctionFusedRGBD with a differentiable camera pose, as GSFunctionFusedPose:
    `apply(pws, shs, alphas, scales, rots, us, Rcw, tcw, twc, cam)` -> (image, depth, alpha,
    depths > 0.2).  The depth plane's gradient reaches the pose through z = (Rcw pw + tcw)[2].
    us_abs (after filter3d) as for GSFunctionFusedRGBD, intrinsics (after us_abs) as for
    GSFunctionFusedPose."""

    @staticmethod
    def forward(ctx, pws, shs, alphas, scales, rots, us, Rcw, tcw, twc, cam, filter3d=None, us_abs=None,
                intrinsics=None):
        return _fused_forward(ctx, True, pws, shs, alphas, scales, rots, us, cam, (Rcw, tcw, twc), filter3d,
                              us_abs=us_abs, intrinsics=intrinsics)

    @staticmethod
    def backward(ctx, dloss_dgammas, dloss_ddepth, dloss_dalpha, _):
        return _fused_backward(ctx, True, True, dloss_dgammas, dloss_ddepth, dloss_dalpha)


class GSFunctionSurfel(torch.autograd.Function):
    """2D Gaussian Splatting (DESIGN 3.15): every Gaussian is a flat disk (surfel) with axes
    scales[:, 0] R e0 and scales[:, 1] R e1 (scales[:, 2] is not read; rots is normalised), drawn
    where the pixel's ray meets it.  `apply(pws, shs, alphas, scales, rots, us, cam)` ->
    (image[3,H,W], depth[H,W], alpha[H,W], normal[3,H,W], depths > 0.2) with
        depth[p] = sum_i w_i(p) z_i(p),  alpha[p] = sum_i w_i(p),  normal[p] = sum_i w_i(p) n_i
    (w = tau alpha'; z_i(p) the camera-frame depth of the ray-splat hit; n_i the camera-frame
    normal facing the camera).  depth is not normalised: depth / alpha is the expected depth.
    Gradients of all four planes reach pws, shs, alphas, scales (column 2: 0), rots and us; us's
    is dL/d of a screen-space shift of the whole surfel, the statistic
    DensityController.update_density_info reads.  A plane the loss does not use is not read in the
    backward (its upstream gradient stays None); with none used, the backward rasterizer is skipped.
    Pinhole cameras only: cam.antialiased, other camera models and cam.grad_exchange are refused,
    and so are filter3d and us_abs."""

    @staticmethod
    def forward(ctx, pws, shs, alphas, scales, rots, us, cam, filter3d=None, us_abs=None):
        from . import ops
        if getattr(cam, "antialiased", False):
            raise ValueError("GSFunctionSurfel has no antialiased mode: cam.antialiased must be False")
        _pinhole_only(cam, "GSFunctionSurfel")
        if getattr(cam, "grad_exchange", None) is not None:
            raise ValueError("GSFunctionSurfel is single-view: cam.grad_exchange must not be set")
        if filter3d is not None:
            raise ValueError("GSFunctionSurfel has no 3D filter: filter3d must be None")
        if us_abs is not None:
            raise ValueError("GSFunctionSurfel has no absolute-gradient statistic: us_abs must be None")
        ctx.set_materialize_grads(False)
        us_, depths, areas, colors, records = ops.surfel_preprocess(
            pws, rots, scales, shs, alphas.reshape(-1), cam.Rcw, cam.tcw, cam.twc, cam.fx, cam.fy, cam.cx, cam.cy,
            cam.width, cam.height)
        image, contrib, final_tau, ranges, gsid, depth, alpha, normal = ops.splat_surfel(
            cam.height, cam.width, us_, depths, areas, records, capacity=True)
        ctx.cam = cam
        ctx.alpha_shape = alphas.shape
        ctx.save_for_backward(pws, shs, scales, rots, records, contrib, final_tau, ranges, gsid)
        return image, depth, alpha, normal, depths > 0.2

    @staticmethod
    def backward(ctx, dloss_dimage, dloss_ddepth, dloss_dalpha, dloss_dnormal, _):
        from . import ops
        cam = ctx.cam
        pws, shs, scales, rots, records, contrib, final_tau, ranges, gsid = ctx.saved_tensors
        rows = ops.splatB_surfel(cam.height, cam.width, records, contrib, final_tau, ranges, gsid,
                                 dloss_dimage, dloss_ddepth, dloss_dalpha, dloss_dnormal)
        dpws, dshs, dalphas, dscales, drots, dus = ops.surfel_preprocessB(
            pws, rots, scales, shs, cam.Rcw, cam.tcw, cam.twc, cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height,
            rows)
        grads = (dpws, dshs, dalphas.reshape(ctx.alpha_shape), dscales, drots, dus)
        return grads + (None,) * (len(ctx.needs_input_grad) - len(grads))


class GSFunctionSurfelGeometry(torch.autograd.Function):
    """GSFunctionSurfel with 2D Gaussian Splatting's geometry terms (DESIGN 3.16).
    `apply(pws, shs, alphas, scales, rots, us, cam, near=0.2, far=100.0)` -> (image, depth, alpha,
    normal, distortion[H,W], median_depth[H,W], depths > 0.2): the first four planes are
    GSFunctionSurfel's (bit for bit), and per pixel, over the surfels in compositing order
    (w = tau alpha', z_i the hit depth, m(z) = far / (far - near) (1 - near / max(z, near))),
        distortion = sum_{j<i} w_i w_j (m_i - m_j)^2      (2DGS's depth-distortion loss, per pixel)
        median_depth = z of the last surfel whose incoming tau > 0.5 (0 where none contributes).
    Unlike 2DGS, m clamps z at near (a hit at or behind the camera would give inf / NaN); below near
    m and its gradient are 0.  All six float planes are differentiable; a plane the loss does not
    use is not read in the backward, and with none used the backward rasterizer is skipped.  With
    no gradient on distortion and median_depth the backward is GSFunctionSurfel's.
    Training loss of 2DGS: L_rgb + lambda_d distortion.mean() + lambda_n L_normal with
    L_normal = (1 - (normal * loss.depth_to_normal(median_depth, cam) * alpha.detach()).sum(0)).mean()
    (2DGS's form, alpha detached; see loss.depth_to_normal).  Refuses cam.antialiased, other camera
    models and cam.grad_exchange, as GSFunctionSurfel does; it takes no filter3d or us_abs, and near /
    far must be numbers with 0 < near < far."""

    @staticmethod
    def forward(ctx, pws, shs, alphas, scales, rots, us, cam, near=0.2, far=100.0):
        from . import ops
        who = "GSFunctionSurfelGeometry"
        if getattr(cam, "antialiased", False):
            raise ValueError("%s has no antialiased mode: cam.antialiased must be False" % who)
        _pinhole_only(cam, who)
        if getattr(cam, "grad_exchange", None) is not None:
            raise ValueError("%s is single-view: cam.grad_exchange must not be set" % who)
        ctx.set_materialize_grads(False)
        us_, depths, areas, colors, records = ops.surfel_preprocess(
            pws, rots, scales, shs, alphas.reshape(-1), cam.Rcw, cam.tcw, cam.twc, cam.fx, cam.fy, cam.cx, cam.cy,
            cam.width, cam.height)
        (image, contrib, final_tau, ranges, gsid, depth, alpha, normal, distortion, median_depth, moments,
         median_contrib) = ops.splat_surfel_geometry(cam.height, cam.width, us_, depths, areas, records, near, far,
                                                     capacity=True)
        ctx.cam, ctx.near, ctx.far = cam, near, far
        ctx.alpha_shape = alphas.shape
        ctx.save_for_backward(pws, shs, scales, rots, records, contrib, final_tau, ranges, gsid, alpha, moments,
                              median_contrib)
        return image, depth, alpha, normal, distortion, median_depth, depths > 0.2

    @staticmethod
    def backward(ctx, dloss_dimage, dloss_ddepth, dloss_dalpha, dloss_dnormal, dloss_ddistortion, dloss_dmedian, _):
        from . import ops
        cam = ctx.cam
        pws, shs, scales, rots, records, contrib, final_tau, ranges, gsid, alpha, moments, median_contrib = \
            ctx.saved_tensors
        rows = ops.splatB_surfel_geometry(cam.height, cam.width, records, contrib, final_tau, ranges, gsid, alpha,
                                          moments, median_contrib, dloss_dimage, dloss_ddepth, dloss_dalpha,
                                          dloss_dnormal, dloss_ddistortion, dloss_dmedian, ctx.near, ctx.far)
        dpws, dshs, dalphas, dscales, drots, dus = ops.surfel_preprocessB(
            pws, rots, scales, shs, cam.Rcw, cam.tcw, cam.twc, cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height,
            rows)
        grads = (dpws, dshs, dalphas.reshape(ctx.alpha_shape), dscales, drots, dus)
        return grads + (None,) * (len(ctx.needs_input_grad) - len(grads))


def _surfel_batch_cams(who, cams, dev):
    """the checks of GSFunctionSurfel / GSFunctionSurfelGeometry per camera, then the batch's own
    (BatchCameras: one width and height for all) -> ops.BatchCameras"""
    from . import ops
    cams = list(cams)
    for c in cams:
        if getattr(c, "antialiased", False):
            raise ValueError("%s has no antialiased mode: cam.antialiased must be False" % who)
        _pinhole_only(c, who)
        if getattr(c, "grad_exchange", None) is not None:
            raise ValueError("%s takes no gradient exchange: cam.grad_exchange must not be set" % who)
    return ops.BatchCameras(cams, dev)


def _surfel_batch_us(us, bc, N):
    if not isinstance(us, torch.Tensor) or tuple(us.shape) != (bc.C, N, 2):
        raise ValueError("us must be a [C, N, 2] tensor (C = %d, N = %d), got %s"
                         % (bc.C, N, tuple(getattr(us, "shape", ()))))


class GSFunctionSurfelBatch(torch.autograd.Function):
    """GSFunctionSurfel for C cameras in one call (DESIGN 3.25): `apply(pws, shs, alphas, scales, rots,
    us, cams)` -> (image[C,3,H,W], depth[C,H,W], alpha[C,H,W], normal[C,3,H,W], mask[C,N]) with frame c
    and mask[c] those GSFunctionSurfel gives for cams[c], bit for bit.  The cameras are pinhole, of one
    width and height (else ValueError), each with its own pose and intrinsics.  us is the [C,N,2]
    dummy whose gradient is each camera's dL/du, so `DensityController.update_density_info(us.grad[c],
    mask[c])` works per camera.  The map gradients are the sums over the cameras, taken in one
    per-surfel pass.  A plane the loss does not use is not read in the backward; with none used the
    backward rasterizer is skipped.  Refuses what GSFunctionSurfel refuses: antialiased cameras, other
    camera models, cam.grad_exchange, filter3d and us_abs."""

    @staticmethod
    def forward(ctx, pws, shs, alphas, scales, rots, us, cams, filter3d=None, us_abs=None):
        from . import ops
        who = "GSFunctionSurfelBatch"
        bc = _surfel_batch_cams(who, cams, pws.device)
        if filter3d is not None:
            raise ValueError("%s has no 3D filter: filter3d must be None" % who)
        if us_abs is not None:
            raise ValueError("%s has no absolute-gradient statistic: us_abs must be None" % who)
        _surfel_batch_us(us, bc, pws.shape[0])
        ctx.set_materialize_grads(False)
        us_, depths, areas, colors, records = ops.surfel_preprocess_batch(pws, rots, scales, shs, alphas.reshape(-1),
                                                                          bc)
        image, contrib, final_tau, ranges, gsid, depth, alpha, normal = ops.splat_surfel_batch(
            bc.height, bc.width, us_, depths, areas, records, capacity=True)
        ctx.bc = bc
        ctx.alpha_shape = alphas.shape
        ctx.save_for_backward(pws, shs, scales, rots, records, contrib, final_tau, ranges, gsid)
        return image, depth, alpha, normal, depths > 0.2

    @staticmethod
    def backward(ctx, dloss_dimage, dloss_ddepth, dloss_dalpha, dloss_dnormal, _):
        from . import ops
        bc = ctx.bc
        pws, shs, scales, rots, records, contrib, final_tau, ranges, gsid = ctx.saved_tensors
        rows = ops.splatB_surfel_batch(bc.height, bc.width, records, contrib, final_tau, ranges, gsid,
                                       dloss_dimage, dloss_ddepth, dloss_dalpha, dloss_dnormal)
        dpws, dshs, dalphas, dscales, drots, dus = ops.surfel_preprocessB_batch(pws, rots, scales, shs, bc, rows)
        grads = (dpws, dshs, dalphas.reshape(ctx.alpha_shape), dscales, drots, dus)
        return grads + (None,) * (len(ctx.needs_input_grad) - len(grads))


class GSFunctionSurfelGeometryBatch(torch.autograd.Function):
    """GSFunctionSurfelGeometry for C cameras in one call (DESIGN 3.25): `apply(pws, shs, alphas, scales,
    rots, us, cams, near=0.2, far=100.0)` -> (image[C,3,H,W], depth[C,H,W], alpha[C,H,W],
    normal[C,3,H,W], distortion[C,H,W], median_depth[C,H,W], mask[C,N]), frame c that of
    GSFunctionSurfelGeometry for cams[c], bit for bit.  Cameras, us and the backward as
    GSFunctionSurfelBatch's; with no gradient on distortion and median_depth the backward is
    GSFunctionSurfelBatch's.  Under torch.no_grad() it is the batched depth renderer of the mesh
    recipe (INTEGRATION.md)."""

    @staticmethod
    def forward(ctx, pws, shs, alphas, scales, rots, us, cams, near=0.2, far=100.0):
        from . import ops
        who = "GSFunctionSurfelGeometryBatch"
        bc = _surfel_batch_cams(who, cams, pws.device)
        _surfel_batch_us(us, bc, pws.shape[0])
        near, far = ops._near_far(near, far)
        ctx.set_materialize_grads(False)
        us_, depths, areas, colors, records = ops.surfel_preprocess_batch(pws, rots, scales, shs, alphas.reshape(-1),
                                                                          bc)
        (image, contrib, final_tau, ranges, gsid, depth, alpha, normal, distortion, median_depth, moments,
         median_contrib) = ops.splat_surfel_geometry_batch(bc.height, bc.width, us_, depths, areas, records, near, far,
                                                           capacity=True)
        ctx.bc, ctx.near, ctx.far = bc, near, far
        ctx.alpha_shape = alphas.shape
        ctx.save_for_backward(pws, shs, scales, rots, records, contrib, final_tau, ranges, gsid, alpha, moments,
                              median_contrib)
        return image, depth, alpha, normal, distortion, median_depth, depths > 0.2

    @staticmethod
    def backward(ctx, dloss_dimage, dloss_ddepth, dloss_dalpha, dloss_dnormal, dloss_ddistortion, dloss_dmedian, _):
        from . import ops
        bc = ctx.bc
        pws, shs, scales, rots, records, contrib, final_tau, ranges, gsid, alpha, moments, median_contrib = \
            ctx.saved_tensors
        rows = ops.splatB_surfel_geometry_batch(bc.height, bc.width, records, contrib, final_tau, ranges, gsid, alpha,
                                                moments, median_contrib, dloss_dimage, dloss_ddepth, dloss_dalpha,
                                                dloss_dnormal, dloss_ddistortion, dloss_dmedian, ctx.near, ctx.far)
        dpws, dshs, dalphas, dscales, drots, dus = ops.surfel_preprocessB_batch(pws, rots, scales, shs, bc, rows)
        grads = (dpws, dshs, dalphas.reshape(ctx.alpha_shape), dscales, drots, dus)
        return grads + (None,) * (len(ctx.needs_input_grad) - len(grads))


@torch.no_grad()
def contribution_stats(pws, shs, alphas, scales, rots, cams, filter3d=None, surfel=False):
    """Per-Gaussian contribution statistics over the views `cams` (DESIGN 3.18), with exactly the
    blending weights w = tau alpha' those views render.  Each camera runs the fused forward the
    training classes run -- 3DGS: ops.preprocess (antialiasing, filter3d and the camera model as in
    GSFunctionFused) and ops.splat; surfel=True: ops.surfel_preprocess and ops.splat_surfel, pinhole
    cameras only, as GSFunctionSurfel -- then the replay (ops.splat_stats / ops.splat_surfel_stats).
    -> dict(weight_sum[N] f32 = sum over views and pixels of w, weight_max[N] f32 = the largest w,
    hit_count[N] i64 = the (view, pixel) pairs with w > 0, views[N] i32 = the cameras in which the
    Gaussian had at least one hit).  The compaction scores built on them are plain torch
    (INTEGRATION.md, "Contribution pruning")."""
    from . import ops
    N, dev = pws.shape[0], pws.device
    weight_sum = torch.zeros(N, dtype=torch.float32, device=dev)
    weight_max = torch.zeros(N, dtype=torch.float32, device=dev)
    hit_count = torch.zeros(N, dtype=torch.int64, device=dev)
    views = torch.zeros(N, dtype=torch.int32, device=dev)
    out = (weight_sum, weight_max, hit_count)
    if surfel and filter3d is not None:
        raise ValueError("surfels have no 3D filter: filter3d must be None")
    if filter3d is not None:
        scales, alphas = ops.filter3d_apply(scales, alphas, filter3d)
    for cam in cams:
        before = hit_count.clone()
        if surfel:
            if getattr(cam, "antialiased", False):
                raise ValueError("surfels have no antialiased mode: cam.antialiased must be False")
            _pinhole_only(cam, "contribution_stats(surfel=True)")
            us, depths, areas, _, records = ops.surfel_preprocess(
                pws, rots, scales, shs, alphas.reshape(-1), cam.Rcw, cam.tcw, cam.twc, cam.fx, cam.fy, cam.cx, cam.cy,
                cam.width, cam.height)
            frame = ops.splat_surfel(cam.height, cam.width, us, depths, areas, records, capacity=True)
            ops.splat_surfel_stats(cam.height, cam.width, records, frame[1], frame[3], frame[4], out=out)
        else:
            aa = bool(getattr(cam, "antialiased", False))
            pre = ops.preprocess(pws, rots, scales, shs, cam.Rcw, cam.tcw, cam.twc, cam.fx, cam.fy, cam.cx, cam.cy,
                                 cam.width, cam.height, alphas=alphas, antialiased=aa, **camera_model_kwargs(cam))
            us, cinv2ds, colors, depths, areas, records = pre[:6]
            drawn = pre[6] if aa else alphas  # the opacities the rasterizer composites
            frame = ops.splat(cam.height, cam.width, us, cinv2ds, drawn, depths, colors, areas, records=records,
                              capacity=True)
            ops.splat_stats(cam.height, cam.width, frame[1], frame[3], frame[4], records=records, out=out)
        views += (hit_count > before).to(torch.int32)
    return dict(weight_sum=weight_sum, weight_max=weight_max, hit_count=hit_count, views=views)
