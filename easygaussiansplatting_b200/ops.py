"""The reference's `gsplatcu` operator surface on top of the C ABI (include/gsplat_b200.h).

Seven functions with the reference's positional signatures, return arity, shapes, dtypes
and in-place side effects (gsplatcu/ext.cpp:10-76, gsplatcu/gausplat.cu): `project`,
`computeCov3D`, `computeCov2D`, `sh2Color`, `inverseCov2D`, `splat`, `splatB`.
torch is used for device memory and the current stream only; all compute is in
libgsplat_b200.so.  Differences from the reference, all deliberate:
  * dtype / device / shape are checked and violations raise (the reference checks nothing);
  * work is enqueued on torch's current stream and nothing device-synchronises except the
    one read of the patch count inside `splat` (the reference syncs the device after every
    kernel, common.cuh:17-25);
  * N == 0 and P <= 1 are handled (SURVEY 8b "degenerate inputs").
"""
import ctypes as C
import math
import numbers

import torch

from . import _lib
from .jacobian_tensor import wrap as _jac

_lib_handle = None


def _L():
    global _lib_handle
    if _lib_handle is None:
        _lib_handle = _lib.load()
    return _lib_handle


def _chk(t, name, dtype=torch.float32, last=None, ndim=None):
    if not isinstance(t, torch.Tensor):
        raise TypeError("%s must be a torch.Tensor" % name)
    if not t.is_cuda:
        raise ValueError("%s must be a CUDA tensor (there is no CPU path)" % name)
    if t.dtype != dtype:
        raise TypeError("%s must be %s, got %s" % (name, dtype, t.dtype))
    if ndim is not None and t.dim() != ndim:
        raise ValueError("%s must have %d dims, got shape %s" % (name, ndim, tuple(t.shape)))
    if last is not None and (t.dim() == 0 or t.shape[-1] != last):
        raise ValueError("%s must have last dim %d, got shape %s" % (name, last, tuple(t.shape)))
    return t.contiguous()


def _same_device(ref, *ts):
    for t in ts:
        if t.device != ref.device:
            raise ValueError("all tensors must be on the same device")


def _shs(shs, N, ref):
    """shs[N, 3k] with k in {1,4,9,16}, on the device of `ref` -> (shs contiguous, k)"""
    shs = _chk(shs, "shs", ndim=2)
    _same_device(ref, shs)
    if shs.shape[0] != N or shs.shape[1] % 3 != 0 or shs.shape[1] // 3 not in (1, 4, 9, 16):
        raise ValueError("shs must be [N, 3k] with k in {1,4,9,16}, got %s" % (tuple(shs.shape),))
    return shs, shs.shape[1] // 3


def _gaussian_map(pws, rots, scales, shs):
    """Checks the per-Gaussian parameters the fused kernels read: float32 CUDA tensors on one
    device, pws[N,3], rots[N,4], scales[N,3], shs[N,3k] with k in {1,4,9,16}.
    -> ((the four tensors, contiguous), N, k)"""
    pws = _chk(pws, "pws", last=3, ndim=2); rots = _chk(rots, "rots", last=4, ndim=2)
    scales = _chk(scales, "scales", last=3, ndim=2)
    _same_device(pws, rots, scales)
    N = pws.shape[0]
    if rots.shape[0] != N or scales.shape[0] != N:
        raise ValueError("pws, rots, scales disagree on N")
    shs, k = _shs(shs, N, pws)
    return (pws, rots, scales, shs), N, k


def _gaussian_params(pws, rots, scales, shs, Rcw, tcw, twc):
    """`_gaussian_map` and the one camera the fused kernels read: Rcw 9, tcw 3 and twc 3 elements
    on the parameters' device.  -> ((the seven tensors, contiguous), N, k)"""
    params, N, k = _gaussian_map(pws, rots, scales, shs)
    Rcw = _chk(Rcw, "Rcw"); tcw = _chk(tcw, "tcw"); twc = _chk(twc, "twc")
    _same_device(params[0], Rcw, tcw, twc)
    if Rcw.numel() != 9 or tcw.numel() != 3 or twc.numel() != 3:
        raise ValueError("Rcw must have 9, tcw and twc 3 elements")
    return params + (Rcw, tcw, twc), N, k


def _scene_args(params, N, k, focal_x, focal_y, center_x, center_y, width, height):
    """The 15 leading arguments of every gsb_preprocess_* entry point, from `_gaussian_params`'
    result (the caller keeps the tensors alive over the call) and the intrinsics"""
    pws, rots, scales, shs, Rcw, tcw, twc = params
    return (N, k, _ptr(pws), _ptr(rots), _ptr(scales), _ptr(shs), _ptr(Rcw), _ptr(tcw), _ptr(twc),
            float(focal_x), float(focal_y), float(center_x), float(center_y), float(width), float(height))


def _per_gaussian(t, name, N, ref):
    """t: a float32 CUDA tensor with N elements on the device of `ref` -> t contiguous"""
    t = _chk(t, name)
    _same_device(ref, t)
    if t.numel() != N:
        raise ValueError("%s must have N elements" % name)
    return t


def _upstream_grads(N, ref, dloss_dus, dloss_dcinv2ds, dloss_dcolors, moments, cinv2ds):
    """Checks the upstream gradients the fused backward reads, float32 CUDA tensors on the device
    of `ref`: moments[N,9] with the forward's cinv2ds[N,3] or, when moments is None, dloss_dus,
    dloss_dcinv2ds, dloss_dcolors (2N, 3N, 3N elements, last dim 2, 3, 3).
    -> (dloss_dus, dloss_dcinv2ds, dloss_dcolors, moments, cinv2ds), contiguous, the unused ones None"""
    if moments is not None:
        moments = _chk(moments, "moments", last=9, ndim=2); cinv2ds = _chk(cinv2ds, "cinv2ds", last=3, ndim=2)
        _same_device(ref, moments, cinv2ds)
        if moments.shape[0] != N or cinv2ds.shape[0] != N:
            raise ValueError("moments / cinv2ds must have N rows")
        return None, None, None, moments, cinv2ds
    gu = _chk(dloss_dus, "dloss_dus", last=2); gc = _chk(dloss_dcinv2ds, "dloss_dcinv2ds", last=3)
    gcol = _chk(dloss_dcolors, "dloss_dcolors", last=3)
    _same_device(ref, gu, gc, gcol)
    if not (gu.numel() == 2 * N and gc.numel() == 3 * N and gcol.numel() == 3 * N):
        raise ValueError("upstream gradients disagree on N")
    return gu, gc, gcol, None, None


def _ptr(t):
    return None if t is None else t.data_ptr()


def _ptrs_if(on, *ts):
    """the pointers of ts when `on`, else none: the arguments only some forms of an entry point take"""
    return [_ptr(t) for t in ts] if on else []


def _stream():
    return torch.cuda.current_stream().cuda_stream


def project(pws, Rcw, tcw, focal_x, focal_y, center_x, center_y, calc_J):
    """ext.cpp:54-61.  -> [us[N,2], pcs[N,3], depths[N]] (+ du_dpcs[N,2,3] if calc_J)"""
    pws = _chk(pws, "pws", last=3, ndim=2)
    Rcw = _chk(Rcw, "Rcw"); tcw = _chk(tcw, "tcw")
    if Rcw.numel() != 9 or tcw.numel() != 3:
        raise ValueError("Rcw must have 9 and tcw 3 elements")
    _same_device(pws, Rcw, tcw)
    N = pws.shape[0]
    o = dict(dtype=torch.float32, device=pws.device)
    us = torch.empty((N, 2), **o); pcs = torch.empty((N, 3), **o); depths = torch.empty((N,), **o)
    J = torch.empty((N, 2, 3), **o) if calc_J else None
    lib = _L()
    with torch.cuda.device(pws.device):
        _lib.check(lib.gsb_project(N, _ptr(pws), _ptr(Rcw), _ptr(tcw), float(focal_x), float(focal_y),
                                   float(center_x), float(center_y), _ptr(us), _ptr(pcs), _ptr(depths),
                                   _ptr(J), _stream()), lib)
    return [us, pcs, depths, _jac(J)] if calc_J else [us, pcs, depths]


def computeCov3D(rots, scales, depths, calc_J):
    """ext.cpp:39-42.  -> [cov3ds[N,6]] (+ dcov3d_drots[N,6,4], dcov3d_dscales[N,6,3])"""
    rots = _chk(rots, "rots", last=4, ndim=2); scales = _chk(scales, "scales", last=3, ndim=2)
    depths = _chk(depths, "depths")
    _same_device(rots, scales, depths)
    N = rots.shape[0]
    if scales.shape[0] != N or depths.numel() != N:
        raise ValueError("rots, scales, depths disagree on N")
    o = dict(dtype=torch.float32, device=rots.device)
    cov = torch.empty((N, 6), **o)
    Jr = torch.empty((N, 6, 4), **o) if calc_J else None
    Js = torch.empty((N, 6, 3), **o) if calc_J else None
    lib = _L()
    with torch.cuda.device(rots.device):
        _lib.check(lib.gsb_compute_cov3d(N, _ptr(rots), _ptr(scales), _ptr(depths), _ptr(cov), _ptr(Jr),
                                         _ptr(Js), _stream()), lib)
    return [cov, _jac(Jr), _jac(Js)] if calc_J else [cov]


def computeCov2D(cov3ds, pcs, Rcw, depths, focal_x, focal_y, width, height, calc_J):
    """ext.cpp:44-52.  -> [cov2ds[N,3]] (+ dcov2d_dcov3ds[N,3,6], dcov2d_dpcs[N,3,3])"""
    cov3ds = _chk(cov3ds, "cov3ds", last=6, ndim=2); pcs = _chk(pcs, "pcs", last=3, ndim=2)
    Rcw = _chk(Rcw, "Rcw"); depths = _chk(depths, "depths")
    _same_device(pcs, cov3ds, Rcw, depths)
    N = pcs.shape[0]
    if cov3ds.shape[0] != N or depths.numel() != N or Rcw.numel() != 9:
        raise ValueError("cov3ds, pcs, depths disagree on N (or Rcw is not 3x3)")
    o = dict(dtype=torch.float32, device=pcs.device)
    cov = torch.empty((N, 3), **o)
    Jc = torch.empty((N, 3, 6), **o) if calc_J else None
    Jp = torch.empty((N, 3, 3), **o) if calc_J else None
    lib = _L()
    with torch.cuda.device(pcs.device):
        _lib.check(lib.gsb_compute_cov2d(N, _ptr(cov3ds), _ptr(pcs), _ptr(Rcw), _ptr(depths),
                                         float(focal_x), float(focal_y), float(width), float(height),
                                         _ptr(cov), _ptr(Jc), _ptr(Jp), _stream()), lib)
    return [cov, _jac(Jc), _jac(Jp)] if calc_J else [cov]


def sh2Color(shs, pws, twc, calc_J):
    """ext.cpp:63-66.  shs[N,3k], k in {1,4,9,16}.
    -> [colors[N,3]] (+ dcolor_dshs[N,1,k], dcolor_dpws[N,3,3])"""
    pws = _chk(pws, "pws", last=3, ndim=2); twc = _chk(twc, "twc")
    _same_device(pws, twc)
    N = pws.shape[0]
    shs, k = _shs(shs, N, pws)
    if twc.numel() != 3:
        raise ValueError("twc must have 3 elements")
    o = dict(dtype=torch.float32, device=pws.device)
    col = torch.empty((N, 3), **o)
    Js = torch.empty((N, 1, k), **o) if calc_J else None
    Jp = torch.empty((N, 3, 3), **o) if calc_J else None
    lib = _L()
    with torch.cuda.device(pws.device):
        _lib.check(lib.gsb_sh2color(N, k, _ptr(shs), _ptr(pws), _ptr(twc), _ptr(col), _ptr(Js), _ptr(Jp),
                                    _stream()), lib)
    return [col, _jac(Js), _jac(Jp)] if calc_J else [col]


def inverseCov2D(cov2ds, depths, calc_J):
    """ext.cpp:34-36.  MUTATES depths (NaN determinant -> -1, kernel.cu:301-305).
    -> [cinv2ds[N,3], areas[N,2] int32] (+ dcinv2d_dcov2ds[N,3,3])"""
    cov2ds = _chk(cov2ds, "cov2ds", last=3, ndim=2); depths = _chk(depths, "depths")
    _same_device(cov2ds, depths)
    N = cov2ds.shape[0]
    if depths.numel() != N:
        raise ValueError("cov2ds and depths disagree on N")
    o = dict(dtype=torch.float32, device=cov2ds.device)
    cinv = torch.empty((N, 3), **o)
    areas = torch.empty((N, 2), dtype=torch.int32, device=cov2ds.device)
    J = torch.empty((N, 3, 3), **o) if calc_J else None
    lib = _L()
    with torch.cuda.device(cov2ds.device):
        _lib.check(lib.gsb_inverse_cov2d(N, _ptr(cov2ds), _ptr(depths), _ptr(cinv), _ptr(areas), _ptr(J),
                                         _stream()), lib)
    return [cinv, areas, _jac(J)] if calc_J else [cinv, areas]


GSB_CAPACITY_EXCEEDED = 2
GSB_STATUS_P_CAP, GSB_STATUS_DEPTH_KEY = 2, 4  # flags of the status word (gsplat_b200.h GSB_STATUS_*)
_CAPACITY = {}  # (device index, H, W, N) -> (P_cap, depth_key_cap) learnt from the previous frame
_STATUS = {}    # device index -> pinned int32[4] for gsb_splat_forward's status read
CAPACITY_STATS = {"capacity_frames": 0, "exact_frames": 0, "outgrown": 0}  # how the frames of `capacity=True` went


def _next_capacity(P, dkmax, headroom=1.25):
    """Bounds for the next frame of the same shape: `headroom` on the patch count, and the key
    width the exact path would pick for a largest depth key of `dkmax`."""
    bits = max(int(dkmax), 1).bit_length()
    return int(P * headroom) + 4096, (1 << bits) - 1


def _decode_status(status):
    """the capacity path's status word [P, largest depth key, flags] (int32 storage) -> unsigned ints"""
    return tuple(int(v) & 0xffffffff for v in status[:3].tolist())


def _bytes(n, dev):
    return torch.empty((n,), dtype=torch.uint8, device=dev)


def _tiles(H, W):
    return ((W + 15) // 16) * ((H + 15) // 16)


def _check_drawn(H, W, ranges, planes, text, frames=None):
    """the per-pixel tensors of a drawn frame, (tensor, channels) in `planes`, against H x W (else
    ValueError(text)), and its patch_range_per_tile against the tile grid.  frames: None, or the C
    of a batch, whose planes and tile ranges hold C frames"""
    Cn = 1 if frames is None else frames
    if any(t.numel() != c * Cn * H * W for t, c in planes):
        raise ValueError(text)
    if ranges.shape[0] != Cn * _tiles(H, W):
        raise ValueError("patch_range_per_tile does not match the %stile grid" % ("" if frames is None else "batch's "))


def _frame_buffers(lib, dev, H, W, N, P, planes, ws_bytes, frames=None):
    """the sort workspace for P patch slots (ws_bytes: the family's workspace query) and splat's
    five outputs, + one plane of each shape in `planes`: float32, or (shape, dtype).  frames: None,
    or the C of a batch: every per-pixel output gets a leading C and the tile ranges C times the rows"""
    lead = () if frames is None else (frames,)
    ws = _bytes(ws_bytes(*lead, N, H, W, P), dev)
    typed = [pl if isinstance(pl[-1], torch.dtype) else (pl, torch.float32) for pl in planes]
    return ws, [torch.empty(lead + (3, H, W), dtype=torch.float32, device=dev),
                torch.empty(lead + (H, W), dtype=torch.int32, device=dev),
                torch.empty(lead + (H, W), dtype=torch.float32, device=dev),
                torch.empty(((frames or 1) * _tiles(H, W), 2), dtype=torch.int32, device=dev),
                torch.empty((P,), dtype=torch.int32, device=dev)] + \
        [torch.empty(lead + tuple(shape), dtype=dtype, device=dev) for shape, dtype in typed]


def _capacity_frame(H, W, us, planes, ws_bytes, forward, P_cap, dk_cap, status, frames=None):
    """Bins, sorts and draws one frame with the sort sized from the bounds (P_cap, dk_cap) through
    forward = (gsb_splat_forward, _rgbd, _enqueue or gsb_splat_surfel_forward, the pointers of its
    frame's own inputs).  planes, ws_bytes, frames: as for `_frame_buffers`.
    -> (False when the frame outgrew a bound, its workspaces, the five outputs with P_cap gsid
    slots + the planes); `status` (pinned int32[4]) receives the status word."""
    lib, N, dev = _L(), us.shape[-2], us.device
    lead = () if frames is None else (frames,)
    bin_ws = _bytes(lib.gsb_splat_bin_batch_workspace_bytes(frames, N) if frames else
                    lib.gsb_splat_bin_workspace_bytes(N), dev)
    ws, out = _frame_buffers(lib, dev, H, W, N, P_cap, planes, ws_bytes, frames)
    entry, inputs = forward
    rc = entry(*lead, H, W, N, *inputs, P_cap, dk_cap, _ptr(bin_ws), bin_ws.numel(), _ptr(ws), ws.numel(),
               *[_ptr(o) for o in out[:5]], status.data_ptr(), *[_ptr(o) for o in out[5:]], _stream())
    if rc != GSB_CAPACITY_EXCEEDED:
        _lib.check(rc, lib)
    return rc == 0, (bin_ws, ws), out


def _frame(H, W, us, depths, areas, planes, ws_bytes, forward, render, capacity, cap_key, frames=None):
    """The one frame driver of `splat`, `splat_rgbd`, `splat_surfel` and `splat_batch`: bins the
    frame (MUTATES depths / areas of what touches no tile) and draws it.  planes, ws_bytes: as for
    `_frame_buffers`; forward, render: (the capacity / the exact entry point, the pointers of the
    frame's own inputs to it).  capacity: size the sort from the bounds learnt for cap_key by the
    previous frame of the same shape; a frame that outgrows them is redone the exact way.
    frames: None, or the C of a batch (us [C, N, 2]): the *_batch entry points, C in front.
    -> (the sort workspace, its patch slots, the outputs with gsid_per_patch of the frame's P)"""
    lib, N, dev = _L(), us.shape[-2], us.device
    lead = () if frames is None else (frames,)
    if capacity and cap_key in _CAPACITY and N > 0:
        P_cap, dk_cap = _CAPACITY[cap_key]
        status = _STATUS.get(dev.index)
        if status is None:
            status = _STATUS[dev.index] = torch.zeros(4, dtype=torch.int32).pin_memory()
        ok, (_, ws), out = _capacity_frame(H, W, us, planes, ws_bytes, forward, P_cap, dk_cap, status, frames)
        if ok:
            CAPACITY_STATS["capacity_frames"] += 1
            P, dkmax, _ = _decode_status(status)
            _CAPACITY[cap_key] = _next_capacity(P, dkmax)
            out[4] = out[4][:P]
            return ws, P_cap, out
        CAPACITY_STATS["outgrown"] += 1
        del _CAPACITY[cap_key]  # outgrown: this frame the exact way (the in-place culls are idempotent)
    bin_ws = _bytes(lib.gsb_splat_bin_batch_workspace_bytes(frames, N) if frames else
                    lib.gsb_splat_bin_workspace_bytes(N), dev)
    P, dkmax = C.c_int64(0), C.c_uint32(0)
    _lib.check((lib.gsb_splat_bin_batch if frames else lib.gsb_splat_bin)(
        *lead, H, W, N, _ptr(us), _ptr(depths), _ptr(areas), _ptr(bin_ws), bin_ws.numel(), C.byref(P),
        C.byref(dkmax), _stream()), lib)
    P = int(P.value)
    ws, out = _frame_buffers(lib, dev, H, W, N, P, planes, ws_bytes, frames)
    if capacity:
        CAPACITY_STATS["exact_frames"] += 1
        _CAPACITY[cap_key] = _next_capacity(P, dkmax.value)
    entry, inputs = render
    _lib.check(entry(*lead, H, W, N, P, dkmax.value, *inputs, _ptr(bin_ws), _ptr(ws), ws.numel(),
                     *[_ptr(o) for o in out], _stream()), lib)
    return ws, P, out


def _attach_records(gsid, records, ws, N, H, W, P_slots, inputs):
    """lets splatB reuse this frame's records: the caller's, or those packed into `ws`, the sort
    workspace of P_slots patches"""
    if gsid.numel() > 0:
        if records is not None:
            _remember_records(gsid, records, 0, inputs)
        else:
            _remember_records(gsid, ws, _L().gsb_splat_records_offset(N, H, W, P_slots), inputs)


def splat(height, width, us, cinv2ds, alphas, depths, colors, areas, records=None, capacity=False):
    """ext.cpp:10-18.  MUTATES depths / areas for Gaussians that touch no tile
    (kernel.cu:114-119).  -> [image[3,H,W], contrib[H,W] i32, final_tau[H,W],
    patch_range_per_tile[T,2] i32, gsid_per_patch[P] i32]
    records (extension): the packed per-Gaussian records `preprocess(..., alphas=...)` wrote;
    the pack pass is then skipped.
    capacity (extension): size the sort from the previous frame of the same shape
    (gsb_splat_forward) instead of reading the patch count back in the middle of the frame; a
    frame that outgrows the bound is transparently redone the exact way."""
    return _splat(height, width, us, cinv2ds, alphas, depths, colors, areas, records, capacity, False)


def splat_rgbd(height, width, us, cinv2ds, alphas, depths, colors, areas, records=None, capacity=False):
    """`splat` (same arguments, same five outputs, bit-identical) plus two [H,W] planes composited
    with the image's weights w = tau alpha':  depth D = sum w z  and  alpha A = sum w,  z = the
    Gaussian's `depths` value.  D is not normalised (the expected depth is D / A); pixels of empty
    tiles get D = A = 0.  -> [image, contrib, final_tau, patch_range_per_tile, gsid_per_patch,
    depth[H,W], alpha[H,W]].  Its backward is `splatB_rgbd`."""
    return _splat(height, width, us, cinv2ds, alphas, depths, colors, areas, records, capacity, True)


def _splat(height, width, us, cinv2ds, alphas, depths, colors, areas, records, capacity, rgbd):
    """the one frame driver of `splat` and `splat_rgbd`"""
    H, W = int(height), int(width)
    if H <= 0 or W <= 0:
        raise ValueError("height and width must be positive")
    us = _chk(us, "us", last=2, ndim=2); cinv2ds = _chk(cinv2ds, "cinv2ds", last=3, ndim=2)
    alphas = _chk(alphas, "alphas"); depths = _chk(depths, "depths")
    colors = _chk(colors, "colors", last=3, ndim=2)
    areas = _chk(areas, "areas", dtype=torch.int32, last=2, ndim=2)
    _same_device(us, cinv2ds, alphas, depths, colors, areas)
    N = us.shape[0]
    if not (cinv2ds.shape[0] == N and alphas.numel() == N and depths.numel() == N
            and colors.shape[0] == N and areas.shape[0] == N):
        raise ValueError("splat inputs disagree on N")
    dev = us.device
    lib = _L()
    if records is not None:
        records = _chk(records, "records", last=12, ndim=2)
        if records.shape[0] != N:
            raise ValueError("records must be [N, 12]")
    # the record cache key: what the records are packed from (depths last: only the RGB-D
    # backward reads the records' depth word, and it looks the records up with depths included)
    inputs = (us, cinv2ds, alphas, colors, depths)
    own = [_ptr(t) for t in (us, cinv2ds, alphas, depths, colors)]
    forward = (lib.gsb_splat_forward_rgbd if rgbd else lib.gsb_splat_forward, own + [_ptr(areas), _ptr(records)])
    render = (lib.gsb_splat_render_rgbd if rgbd else lib.gsb_splat_render, own + [_ptr(records)])
    # the workspaces are consumed by kernels already enqueued on the current stream; the caching
    # allocator only reuses them for later work on the same stream
    with torch.cuda.device(dev):
        ws, P_slots, out = _frame(H, W, us, depths, areas, [(H, W)] * 2 if rgbd else [], lib.gsb_splat_workspace_bytes,
                                  forward, render, capacity, (dev.index, H, W, N))
        _attach_records(out[4], records, ws, N, H, W, P_slots, inputs)
    return out


# The forward leaves the packed per-Gaussian records in its workspace (or got them from
# `preprocess`); splatB can reuse them instead of packing the same records again.  The handle
# travels ON the gsid_per_patch tensor `splat` returns (an attribute of that tensor object; it
# survives autograd's save_for_backward), so identity is never inferred from addresses the
# caching allocator may hand out again, and the workspace lives exactly as long as that tensor.
# The inputs must still be the very tensors the forward saw, unmodified (data_ptr + torch's
# in-place version counter); writes that bypass the counter (`.data`, foreign kernels) are the
# caller's to announce with `forget_records(gsid)`.  The key covers us, cinv2ds, alphas, colors
# and depths; `splatB` matches the first four (its kernel never reads the depth word), `splatB_rgbd`
# all five, so it never uses records whose depth word is stale.
_RECORDS_ATTR = "_gsb_records"


def _input_key(inputs):
    try:
        return tuple((t.data_ptr(), t._version) for t in inputs)
    except RuntimeError:  # inference tensors have no version counter: never cache
        return None


def _remember_records(gsid, ws, offset, inputs):
    key = _input_key(inputs)
    if key is not None:
        setattr(gsid, _RECORDS_ATTR, (ws, offset, key, gsid.data_ptr(), gsid.numel()))


def _cached_records(gsid, inputs):
    h = getattr(gsid, _RECORDS_ATTR, None)
    if h is None:
        return None
    ws, offset, key, gptr, P = h
    want = _input_key(inputs)
    if gptr != gsid.data_ptr() or P != gsid.numel() or want is None or key is None or key[:len(want)] != want:
        return None
    return ws.data_ptr() + offset


def forget_records(gsid):
    """Drop the packed records `splat` attached to its gsid_per_patch output (frees the forward
    workspace early; splatB then packs the records again)."""
    if hasattr(gsid, _RECORDS_ATTR):
        delattr(gsid, _RECORDS_ATTR)


def clear_record_cache():
    """Kept for callers of the round-1 API: there is no global cache any more (see above)."""


def splatB(height, width, us, cinv2ds, alphas, depths, colors, contrib, final_tau,
           patch_range_per_tile, gsid_per_patch, dloss_dgammas, moments_only=False, records=None, absgrad=False):
    """ext.cpp:20-32.  -> [dloss_dus[N,1,2], dloss_dcinv2ds[N,1,3], dloss_dalphas[N,1,1],
    dloss_dcolors[N,1,3]]   (`depths` is accepted and unused, as in the reference)
    moments_only (extension): -> the raw moment rows [N,9] for `preprocessB(..., moments=...)`;
    the conversion pass to the four tensors is skipped.
    records (extension): the forward's packed per-Gaussian records [N,12] (what `splat` was given,
    or its own); they are used as they are instead of those `splat` attached to gsid_per_patch,
    and nothing is re-packed.
    absgrad (extension; AbsGS): dloss_dus_abs[N,2], the per-pixel absolute sums of dL/du
    (gsb_splat_backward_abs), is appended to what the call returns otherwise; every other output
    is the same."""
    return _splatB(height, width, us, cinv2ds, alphas, depths, colors, contrib, final_tau, patch_range_per_tile,
                   gsid_per_patch, dloss_dgammas, None, None, moments_only, records, absgrad)


def splatB_rgbd(height, width, us, cinv2ds, alphas, depths, colors, contrib, final_tau, patch_range_per_tile,
                gsid_per_patch, dloss_dgammas, dloss_ddepth, dloss_dalpha, moments_only=False, records=None,
                absgrad=False):
    """Backward of `splat_rgbd`: `splatB`'s arguments plus dloss_ddepth[H,W] and dloss_dalpha[H,W]
    (dL/dD, dL/dA); `depths` is read (the records' depth words).
    -> [dloss_dus, dloss_dcinv2ds, dloss_dalphas, dloss_dcolors] as `splatB`, + dloss_ddepths[N]
    (dL/dz of every Gaussian's `depths` value); with moments_only: [moments[N,9], dloss_ddepths]
    for `preprocessB(..., moments=..., dloss_ddepths=...)`.
    records: as for `splatB`; they must carry z, as those `preprocess(..., alphas=...)` returns do.
    Records `splat` / `splat_rgbd` attached to gsid_per_patch are used only while `depths` is
    unchanged too; otherwise they are re-packed from the arguments.
    absgrad: as for `splatB`, appended last (the upstream gradient of all three planes enters it)."""
    return _splatB(height, width, us, cinv2ds, alphas, depths, colors, contrib, final_tau, patch_range_per_tile,
                   gsid_per_patch, dloss_dgammas, dloss_ddepth, dloss_dalpha, moments_only, records, absgrad)


def _splatB(height, width, us, cinv2ds, alphas, depths, colors, contrib, final_tau, patch_range_per_tile,
            gsid_per_patch, dloss_dgammas, dloss_ddepth, dloss_dalpha, moments_only, records, absgrad=False):
    """`splatB`, or `splatB_rgbd` when dloss_ddepth is given; absgrad: the _abs entry points"""
    rgbd = dloss_ddepth is not None
    H, W = int(height), int(width)
    us = _chk(us, "us", last=2, ndim=2); cinv2ds = _chk(cinv2ds, "cinv2ds", last=3, ndim=2)
    alphas = _chk(alphas, "alphas"); colors = _chk(colors, "colors", last=3, ndim=2)
    contrib = _chk(contrib, "contrib", dtype=torch.int32); final_tau = _chk(final_tau, "final_tau")
    ranges = _chk(patch_range_per_tile, "patch_range_per_tile", dtype=torch.int32, last=2)
    gsid = _chk(gsid_per_patch, "gsid_per_patch", dtype=torch.int32)
    dl = _chk(dloss_dgammas, "dloss_dgammas")
    _same_device(us, cinv2ds, alphas, colors, contrib, final_tau, ranges, gsid, dl)
    N = us.shape[0]
    _check_drawn(H, W, ranges, ((contrib, 1), (final_tau, 1), (dl, 3)),
                 "contrib / final_tau / dloss_dgammas do not match height x width")
    if not (cinv2ds.shape[0] == N and alphas.numel() == N and colors.shape[0] == N):
        raise ValueError("splatB inputs disagree on N")
    if rgbd:
        depths = _chk(depths, "depths")
        dloss_ddepth = _chk(dloss_ddepth, "dloss_ddepth"); dloss_dalpha = _chk(dloss_dalpha, "dloss_dalpha")
        _same_device(us, depths, dloss_ddepth, dloss_dalpha)
        if depths.numel() != N:
            raise ValueError("splatB_rgbd inputs disagree on N")
        if dloss_ddepth.numel() != H * W or dloss_dalpha.numel() != H * W:
            raise ValueError("dloss_ddepth / dloss_dalpha do not match height x width")
    if records is not None:
        records = _chk(records, "records", last=12, ndim=2)
        _same_device(us, records)
        if records.shape[0] != N:
            raise ValueError("records must be [N, 12]")
    P = gsid.numel()
    dev = us.device
    o = dict(dtype=torch.float32, device=dev)
    if moments_only:
        du = dc = da = dcol = None
        moments = torch.empty((N, 9), **o)
    else:
        du = torch.empty((N, 1, 2), **o); dc = torch.empty((N, 1, 3), **o)
        da = torch.empty((N, 1, 1), **o); dcol = torch.empty((N, 1, 3), **o)
        moments = None
    ddepths = torch.empty((N,), **o) if rgbd else None
    dabs = torch.empty((N, 2), **o) if absgrad else None
    lib = _L()
    with torch.cuda.device(dev):
        if records is not None:
            recs = records.data_ptr()
        else:
            key = (us, cinv2ds, alphas, colors, depths) if rgbd else (us, cinv2ds, alphas, colors)
            recs = _cached_records(gsid, key) if P > 0 else None
        # with cached records only the [N,9] moment rows are needed from the workspace
        ws = _bytes(lib.gsb_splat_backward_workspace_bytes(N, H, W, 0 if recs else P), dev)
        # gsb_splat_backward{,_rgbd}{,_abs}: the RGB-D forms take depths, the two planes' gradients and
        # dloss_ddepths, the _abs forms dloss_dus_abs last
        entry = getattr(lib, "gsb_splat_backward" + ("_rgbd" if rgbd else "") + ("_abs" if absgrad else ""))
        _lib.check(entry(H, W, N, P, _ptr(us), _ptr(cinv2ds), _ptr(alphas), _ptr(colors), *_ptrs_if(rgbd, depths),
                         _ptr(contrib), _ptr(final_tau), _ptr(ranges), _ptr(gsid), _ptr(dl),
                         *_ptrs_if(rgbd, dloss_ddepth, dloss_dalpha), recs, _ptr(ws), ws.numel(), _ptr(du), _ptr(dc),
                         _ptr(da), _ptr(dcol), _ptr(moments), *_ptrs_if(rgbd, ddepths), *_ptrs_if(absgrad, dabs),
                         _stream()), lib)
    if moments_only:
        out = [moments, ddepths] if rgbd else moments
    else:
        # tagged so that the reference's `dloss_d* @ jacobian` chain takes the streaming matmul
        out = [_jac(du), _jac(dc), _jac(da), _jac(dcol)]
        out = out + [ddepths] if rgbd else out
    if not absgrad:
        return out
    return (out if isinstance(out, list) else [out]) + [dabs]


# ---------------------------------------------------------------------------------------
# Batched rendering (extension, DESIGN 3.21): C cameras of one image size, camera model and
# antialiasing mode in one call.  The per-Gaussian kernels read each Gaussian's rows once for all
# C cameras; the C frames are binned, sorted and drawn as one tall frame.  Record c N + n is
# Gaussian n seen by camera c; per-record outputs are [C, N, ...], per-pixel ones [C, ..., H, W].
BATCH_MAX_CAMERAS = 64     # cameras per call (GSB_BATCH_MAX_CAMERAS)
BATCH_INTRINSICS_ROW = 8   # fx, fy, cx, cy, k[4] (GSB_BATCH_INTRINSICS_ROW)


class BatchCameras:
    """The cameras of one batch, checked on the host: poses [C, 15] (Rcw row-major, tcw, twc) on the
    device, intrinsics [C, 8] (fx, fy, cx, cy, k[4]) on the host, and what they share: width,
    height, antialiased, camera_model.  Cameras that disagree on a shared field are a ValueError.
    poses: None, or a [C, 15] float32 tensor on `device` that replaces the cameras' own Rcw, tcw, twc
    (DESIGN 3.22: the poses being optimised; read as a constant, never copied to the host)."""

    def __init__(self, cams, device, poses=None):
        from .gsfunction import camera_model_kwargs
        cams = list(cams)
        if not 1 <= len(cams) <= BATCH_MAX_CAMERAS:
            raise ValueError("a batch takes 1 to %d cameras, got %d" % (BATCH_MAX_CAMERAS, len(cams)))
        c0 = cams[0]
        self.width, self.height = int(c0.width), int(c0.height)
        self.antialiased = bool(getattr(c0, "antialiased", False))
        self.camera_model = getattr(c0, "camera_model", "pinhole")
        rows, own = [], []
        for k, c in enumerate(cams):
            shared = (int(c.width), int(c.height), bool(getattr(c, "antialiased", False)),
                      getattr(c, "camera_model", "pinhole"))
            if shared != (self.width, self.height, self.antialiased, self.camera_model):
                raise ValueError("camera %d: the cameras of a batch share width, height, antialiased and "
                                 "camera_model, got %s and %s" % (k, shared, (self.width, self.height,
                                                                            self.antialiased, self.camera_model)))
            _, lk = camera_model_args(**camera_model_kwargs(c))
            rows.append([float(c.fx), float(c.fy), float(c.cx), float(c.cy)] + list(lk))
            if poses is not None:
                continue
            pose = [torch.as_tensor(t).detach().reshape(-1).to(device=device, dtype=torch.float32)
                    for t in (c.Rcw, c.tcw, c.twc)]
            if [t.numel() for t in pose] != [9, 3, 3]:
                raise ValueError("camera %d: Rcw must have 9, tcw and twc 3 elements" % k)
            own.append(torch.cat(pose))
        self.C = len(cams)
        self.model_id = _CAMERA_MODEL_ID[self.camera_model]
        if poses is None:
            self.poses = torch.stack(own).contiguous()
        else:
            if not isinstance(poses, torch.Tensor) or tuple(poses.shape) != (self.C, 15) or \
                    poses.dtype != torch.float32:
                raise ValueError("poses must be a [C, 15] float32 tensor (C = %d), got %s"
                                 % (self.C, tuple(getattr(poses, "shape", ()))))
            if poses.device != torch.device(device):
                raise ValueError("poses must be on %s, got %s" % (device, poses.device))
            self.poses = poses.detach().contiguous()
        self.intrinsics = torch.tensor(rows, dtype=torch.float32)

    def args(self):
        """poses, intrinsics, camera_model, width, height as the batch entry points take them"""
        return (_ptr(self.poses), self.intrinsics.data_ptr(), self.model_id, float(self.width), float(self.height))


def _batch_cams(cams, device):
    return cams if isinstance(cams, BatchCameras) else BatchCameras(cams, device)


def preprocess_batch(pws, rots, scales, shs, cams, alphas):
    """`preprocess(..., alphas=alphas, antialiased=..., camera_model=...)` for C cameras at once
    (gsb_preprocess_forward_batch).  cams: a list of `gsfunction.Camera` (or a `BatchCameras`)
    sharing width, height, antialiased and camera_model.  -> [us[C,N,2], cinv2ds[C,N,3],
    colors[C,N,3], depths[C,N], areas[C,N,2] int32, records[C N, 12]] + [alphas_eff[C,N]] when
    antialiased; camera c's rows are the bits `preprocess` gives for camera c alone."""
    (pws, rots, scales, shs), N, k = _gaussian_map(pws, rots, scales, shs)
    bc = _batch_cams(cams, pws.device)
    alphas = _per_gaussian(alphas, "alphas", N, pws)
    Cn = bc.C
    o = dict(dtype=torch.float32, device=pws.device)
    us = torch.empty((Cn, N, 2), **o); cinv = torch.empty((Cn, N, 3), **o); col = torch.empty((Cn, N, 3), **o)
    depths = torch.empty((Cn, N), **o); areas = torch.empty((Cn, N, 2), dtype=torch.int32, device=pws.device)
    records = torch.empty((Cn * N, 12), **o)
    alphas_eff = torch.empty((Cn, N), **o) if bc.antialiased else None
    lib = _L()
    with torch.cuda.device(pws.device):
        _lib.check(lib.gsb_preprocess_forward_batch(
            Cn, N, k, _ptr(pws), _ptr(rots), _ptr(scales), _ptr(shs), *bc.args(), _ptr(us), _ptr(cinv), _ptr(col),
            _ptr(depths), _ptr(areas), _ptr(alphas), _ptr(records), _ptr(alphas_eff), _stream()), lib)
    out = [us, cinv, col, depths, areas, records]
    return out + [alphas_eff] if bc.antialiased else out


def preprocessB_batch(pws, rots, scales, shs, cams, moments, cinv2ds, dloss_ddepths=None, alphas=None,
                      camera_grad=False, pose_only=False, intrinsics_grad=False):
    """Backward of `preprocess_batch` from the moment rows [C N, 9] of `splatB_batch` and the
    forward's cinv2ds [C,N,3] (gsb_preprocess_backward_batch): the C cameras' contributions summed
    in fp32 registers in camera order.  dloss_ddepths [C N]: the RGB-D term; alphas [N]: the raw
    opacities, required when the cameras are antialiased.
    -> [dloss_dpws[N,3], dloss_dshs[N,3k], dloss_dscales[N,3], dloss_drots[N,4], dloss_dus[C,N,2]
    (per camera), dloss_dalphas[N]]
    camera_grad (DESIGN 3.22, gsb_preprocess_backward_batch_pose): one more output follows, the
    camera gradients (dRcws[C,3,3], dtcws[C,3], dtwcs[C,3]) -- views of one [C, 15] tensor; row c is
    what `preprocessB(..., camera_grad=True)` gives for camera c alone.  The per-Gaussian outputs are
    the same bits as without it.  pose_only (with camera_grad): the map is frozen; the six
    per-Gaussian outputs are not computed and come back as None.
    intrinsics_grad (with camera_grad; DESIGN 3.23, gsb_preprocess_backward_batch_intrinsics): one more
    output follows, dintrinsics[C, 8] in the layout of BatchCameras.intrinsics; row c is what
    `preprocessB(..., intrinsics_grad=True)` gives for camera c alone."""
    if pose_only and not camera_grad:
        raise ValueError("pose_only=True needs camera_grad=True")
    if intrinsics_grad and not camera_grad:
        raise ValueError("intrinsics_grad=True needs camera_grad=True")
    (pws, rots, scales, shs), N, k = _gaussian_map(pws, rots, scales, shs)
    bc = _batch_cams(cams, pws.device)
    Cn = bc.C
    moments = _chk(moments, "moments", last=9); cinv2ds = _chk(cinv2ds, "cinv2ds", last=3)
    _same_device(pws, moments, cinv2ds)
    if moments.numel() != 9 * Cn * N or cinv2ds.numel() != 3 * Cn * N:
        raise ValueError("moments / cinv2ds must have C N rows")
    if dloss_ddepths is not None:
        dloss_ddepths = _per_gaussian(dloss_ddepths, "dloss_ddepths", Cn * N, pws)
    if bc.antialiased and alphas is None:
        raise ValueError("antialiased cameras need the raw alphas")
    alphas = _per_gaussian(alphas, "alphas", N, pws) if bc.antialiased else None
    o = dict(dtype=torch.float32, device=pws.device)
    if pose_only:
        gpw = gsh = gs = gq = dus = dal = None
    else:
        gpw = torch.empty((N, 3), **o); gsh = torch.empty((N, 3 * k), **o)
        gs = torch.empty((N, 3), **o); gq = torch.empty((N, 4), **o)
        dus = torch.empty((Cn, N, 2), **o); dal = torch.empty((N,), **o)
    lib = _L()
    with torch.cuda.device(pws.device):
        args = (Cn, N, k, _ptr(pws), _ptr(rots), _ptr(scales), _ptr(shs), *bc.args(), _ptr(moments), _ptr(cinv2ds),
                _ptr(dloss_ddepths), _ptr(alphas), _ptr(gpw), _ptr(gsh), _ptr(gs), _ptr(gq), _ptr(dus), _ptr(dal))
        if intrinsics_grad:
            gcam = torch.empty((Cn, 15), **o)
            gint = torch.empty((Cn, BATCH_INTRINSICS_ROW), **o)
            ws_bytes = int(lib.gsb_preprocess_backward_batch_intrinsics_workspace_bytes(Cn, N))
            ws = torch.empty((max(ws_bytes, 16),), dtype=torch.uint8, device=pws.device)
            _lib.check(lib.gsb_preprocess_backward_batch_intrinsics(*args, _ptr(gcam), _ptr(gint), _ptr(ws), ws_bytes,
                                                                    _stream()), lib)
        elif camera_grad:
            gcam = torch.empty((Cn, 15), **o)
            ws_bytes = int(lib.gsb_preprocess_backward_batch_pose_workspace_bytes(Cn, N))
            ws = torch.empty((max(ws_bytes, 16),), dtype=torch.uint8, device=pws.device)
            _lib.check(lib.gsb_preprocess_backward_batch_pose(*args, _ptr(gcam), _ptr(ws), ws_bytes, _stream()), lib)
        else:
            _lib.check(lib.gsb_preprocess_backward_batch(*args, _stream()), lib)
    out = [gpw, gsh, gs, gq, dus, dal]
    if camera_grad:
        out.append((gcam[:, :9].view(Cn, 3, 3), gcam[:, 9:12], gcam[:, 12:15]))
    if intrinsics_grad:
        out.append(gint)
    return out


def _batch_frame_inputs(us, cinv2ds, alphas, depths, colors, records):
    """the [C, N, ...] inputs of a batch frame, checked -> (C, N, the inputs contiguous).  alphas:
    [C, N] (the drawn opacities per camera), or [N] when records are given (then not read)."""
    us = _chk(us, "us", last=2, ndim=3)
    Cn, N = us.shape[0], us.shape[1]
    cinv2ds = _chk(cinv2ds, "cinv2ds", last=3, ndim=3); colors = _chk(colors, "colors", last=3, ndim=3)
    depths = _chk(depths, "depths"); alphas = _chk(alphas, "alphas")
    _same_device(us, cinv2ds, colors, depths, alphas)
    if not (tuple(cinv2ds.shape[:2]) == (Cn, N) and tuple(colors.shape[:2]) == (Cn, N)
            and depths.numel() == Cn * N):
        raise ValueError("batch frame inputs disagree on C, N")
    if alphas.numel() != Cn * N and not (records is not None and alphas.numel() == N):
        raise ValueError("alphas must be [C, N] (or [N] with records)")
    if records is not None:
        records = _chk(records, "records", last=12, ndim=2)
        _same_device(us, records)
        if records.shape[0] != Cn * N:
            raise ValueError("records must be [C N, 12]")
    return Cn, N, us, cinv2ds, alphas, depths, colors, records


def splat_batch(height, width, us, cinv2ds, alphas, depths, colors, areas, records=None, capacity=False,
                rgbd=False):
    """`splat` (or, rgbd, `splat_rgbd`) of C frames of height x width at once, binned and drawn as
    one tall frame (gsb_splat_render_batch / gsb_splat_forward_batch and their _rgbd forms).
    Inputs are `preprocess_batch`'s [C, N, ...] outputs; MUTATES depths / areas of records that
    touch no tile.  -> [image[C,3,H,W], contrib[C,H,W] i32, final_tau[C,H,W],
    patch_range_per_tile[C T, 2] i32, gsid_per_patch[P] i32 (record ids c N + n)]
    + [depth[C,H,W], alpha[C,H,W]] with rgbd.  Frame c is the single frame of camera c, bit for bit.
    records, capacity: as for `splat`."""
    H, W = int(height), int(width)
    if H <= 0 or W <= 0:
        raise ValueError("height and width must be positive")
    Cn, N, us, cinv2ds, alphas, depths, colors, records = _batch_frame_inputs(us, cinv2ds, alphas, depths, colors,
                                                                              records)
    areas = _chk(areas, "areas", dtype=torch.int32, last=2, ndim=3)
    if tuple(areas.shape[:2]) != (Cn, N):
        raise ValueError("areas must be [C, N, 2]")
    if records is None and alphas.numel() != Cn * N:
        raise ValueError("alphas must be [C, N] without records")
    dev = us.device
    lib = _L()
    own = [_ptr(t) for t in (us, cinv2ds, alphas, depths, colors)]
    sfx = "_rgbd" if rgbd else ""
    forward = (getattr(lib, "gsb_splat_forward_batch" + sfx), own + [_ptr(areas), _ptr(records)])
    render = (getattr(lib, "gsb_splat_render_batch" + sfx), own + [_ptr(records)])
    with torch.cuda.device(dev):
        _, _, out = _frame(H, W, us, depths, areas, [(H, W)] * 2 if rgbd else [], lib.gsb_splat_batch_workspace_bytes,
                           forward, render, capacity, ("batch", dev.index, Cn, H, W, N), frames=Cn)
    return out


def splatB_batch(height, width, us, cinv2ds, alphas, depths, colors, contrib, final_tau, patch_range_per_tile,
                 gsid_per_patch, dloss_dgammas, dloss_ddepth=None, dloss_dalpha=None, records=None):
    """Backward of `splat_batch` (gsb_splat_backward_batch, or _rgbd when dloss_ddepth[C,H,W] and
    dloss_dalpha[C,H,W] are given): dloss_dgammas [C,3,H,W] -> the moment rows [C N, 9] for
    `preprocessB_batch` (+ dloss_ddepths [C N] with RGB-D).  records: the forward's [C N, 12], or
    None (re-packed from us, cinv2ds, alphas [C,N], colors and depths)."""
    rgbd = dloss_ddepth is not None
    H, W = int(height), int(width)
    Cn, N, us, cinv2ds, alphas, depths, colors, records = _batch_frame_inputs(us, cinv2ds, alphas, depths, colors,
                                                                              records)
    contrib = _chk(contrib, "contrib", dtype=torch.int32); final_tau = _chk(final_tau, "final_tau")
    ranges = _chk(patch_range_per_tile, "patch_range_per_tile", dtype=torch.int32, last=2)
    gsid = _chk(gsid_per_patch, "gsid_per_patch", dtype=torch.int32)
    dl = _chk(dloss_dgammas, "dloss_dgammas")
    _same_device(us, contrib, final_tau, ranges, gsid, dl)
    _check_drawn(H, W, ranges, ((contrib, 1), (final_tau, 1), (dl, 3)),
                 "contrib / final_tau / dloss_dgammas do not match C x height x width", frames=Cn)
    if rgbd:
        dloss_ddepth = _chk(dloss_ddepth, "dloss_ddepth"); dloss_dalpha = _chk(dloss_dalpha, "dloss_dalpha")
        _same_device(us, dloss_ddepth, dloss_dalpha)
        if dloss_ddepth.numel() != Cn * H * W or dloss_dalpha.numel() != Cn * H * W:
            raise ValueError("dloss_ddepth / dloss_dalpha do not match C x height x width")
    P = gsid.numel()
    dev = us.device
    moments = torch.empty((Cn * N, 9), dtype=torch.float32, device=dev)
    ddepths = torch.empty((Cn * N,), dtype=torch.float32, device=dev) if rgbd else None
    lib = _L()
    with torch.cuda.device(dev):
        ws = _bytes(lib.gsb_splat_backward_batch_workspace_bytes(Cn, N, H, W, 0 if records is not None else P), dev)
        entry = getattr(lib, "gsb_splat_backward_batch" + ("_rgbd" if rgbd else ""))
        _lib.check(entry(Cn, H, W, N, P, _ptr(us), _ptr(cinv2ds), _ptr(alphas), _ptr(colors), *_ptrs_if(rgbd, depths),
                         _ptr(contrib), _ptr(final_tau), _ptr(ranges), _ptr(gsid), _ptr(dl),
                         *_ptrs_if(rgbd, dloss_ddepth, dloss_dalpha), _ptr(records), _ptr(ws), ws.numel(),
                         _ptr(moments), *_ptrs_if(rgbd, ddepths), _stream()), lib)
    return [moments, ddepths] if rgbd else moments


# ---------------------------------------------------------------------------------------
# Feature rendering (extension): per-Gaussian feature vectors composited with the image's weights.
def _feature_frame(height, width, features, contrib, patch_range_per_tile, gsid_per_patch, records, us, cinv2ds,
                   alphas, colors):
    """the checks both feature operators make -> (H, W, N, D, P, features, contrib, ranges, gsid,
    the record pointer or None, (us, cinv2ds, alphas, colors) for a re-pack), on the device of features"""
    H, W = int(height), int(width)
    if H <= 0 or W <= 0:
        raise ValueError("height and width must be positive")
    features = _chk(features, "features", ndim=2)
    if features.shape[1] < 1:
        raise ValueError("features must be [N, D] with D >= 1, got shape %s" % (tuple(features.shape),))
    N, D = features.shape
    contrib = _chk(contrib, "contrib", dtype=torch.int32)
    ranges = _chk(patch_range_per_tile, "patch_range_per_tile", dtype=torch.int32, last=2)
    gsid = _chk(gsid_per_patch, "gsid_per_patch", dtype=torch.int32)
    _same_device(features, contrib, ranges, gsid)
    _check_drawn(H, W, ranges, ((contrib, 1),), "contrib does not match height x width")
    P = gsid.numel()
    attrs = (None,) * 4
    recs = None
    if records is not None:
        records = _chk(records, "records", last=12, ndim=2)
        _same_device(features, records)
        if records.shape[0] != N:
            raise ValueError("records must be [N, 12]")
        recs = records.data_ptr()
    elif P > 0:
        if any(x is None for x in (us, cinv2ds, alphas, colors)):
            raise ValueError("give the forward's records, or us, cinv2ds, alphas and colors to find or re-pack them")
        us = _chk(us, "us", last=2, ndim=2); cinv2ds = _chk(cinv2ds, "cinv2ds", last=3, ndim=2)
        alphas = _chk(alphas, "alphas"); colors = _chk(colors, "colors", last=3, ndim=2)
        _same_device(features, us, cinv2ds, alphas, colors)
        if not (us.shape[0] == N and cinv2ds.shape[0] == N and alphas.numel() == N and colors.shape[0] == N):
            raise ValueError("features, us, cinv2ds, alphas and colors disagree on N")
        attrs = (us, cinv2ds, alphas, colors)
        recs = _cached_records(gsid, attrs)  # those `splat` attached, while its inputs are unchanged
    return H, W, N, D, P, features, contrib, ranges, gsid, recs, attrs


def splat_features(height, width, features, contrib, patch_range_per_tile, gsid_per_patch, records=None, us=None,
                   cinv2ds=None, alphas=None, colors=None):
    """The feature map of a frame `splat` (or `splat_rgbd`) drew (gsb_splat_features):
        feature_map[c, p] = sum_i w_i(p) features[i, c],   w = tau alpha', the image's weights
    features[N, D] (any D >= 1; f = the colours gives the image's bits).  contrib,
    patch_range_per_tile, gsid_per_patch: that frame's outputs.  records: the forward's packed
    records [N,12] (`preprocess(..., alphas=...)`'s, as given to `splat`); otherwise those `splat`
    attached to gsid_per_patch are used while us, cinv2ds, alphas and colors (then required) are
    the tensors it saw, unchanged, and re-packed from them if not.  -> feature_map[D, H, W]
    (0 on tiles without patches).  Its backward is `splatB_features`."""
    H, W, N, D, P, features, contrib, ranges, gsid, recs, attrs = _feature_frame(
        height, width, features, contrib, patch_range_per_tile, gsid_per_patch, records, us, cinv2ds, alphas, colors)
    dev = features.device
    out = torch.empty((D, H, W), dtype=torch.float32, device=dev)
    lib = _L()
    with torch.cuda.device(dev):
        ws = _bytes(lib.gsb_splat_features_workspace_bytes(N, H, W, 0 if recs else P), dev)
        _lib.check(lib.gsb_splat_features(H, W, N, P, D, *[_ptr(a) for a in attrs], _ptr(features), recs, _ptr(contrib),
                                          _ptr(ranges), _ptr(gsid), _ptr(ws), ws.numel(), _ptr(out), _stream()), lib)
    return out


def splatB_features(height, width, features, contrib, final_tau, patch_range_per_tile, gsid_per_patch,
                    dloss_dfeature_map, moments=None, records=None, us=None, cinv2ds=None, alphas=None, colors=None):
    """Backward of `splat_features` (gsb_splat_features_backward): dloss_dfeature_map[D, H, W] ->
    (moments[N, 9], dloss_dfeatures[N, D]).  The feature map's dL/dalpha' enters moment rows 0-5,
    the form `splatB(..., moments_only=True)` returns, so `preprocessB(..., moments=...)` turns
    them into the geometry and opacity gradients.  moments: None (fresh rows, rows 6-8 zero), or
    such rows (contiguous float32 [N, 9]) to ADD to in place -- chain it after
    `splatB(..., moments_only=True)` / `splatB_rgbd` for a loss on both maps.  records, us,
    cinv2ds, alphas, colors: as for `splat_features`."""
    H, W, N, D, P, features, contrib, ranges, gsid, recs, attrs = _feature_frame(
        height, width, features, contrib, patch_range_per_tile, gsid_per_patch, records, us, cinv2ds, alphas, colors)
    final_tau = _chk(final_tau, "final_tau")
    dl = _chk(dloss_dfeature_map, "dloss_dfeature_map")
    _same_device(features, final_tau, dl)
    if final_tau.numel() != H * W or dl.numel() != D * H * W:
        raise ValueError("final_tau / dloss_dfeature_map do not match D x height x width")
    dev = features.device
    if moments is None:
        moments = torch.zeros((N, 9), dtype=torch.float32, device=dev)
    elif not (isinstance(moments, torch.Tensor) and moments.is_cuda and moments.dtype == torch.float32 and
              tuple(moments.shape) == (N, 9) and moments.is_contiguous() and moments.device == dev):
        raise ValueError("moments must be a contiguous float32 [N, 9] tensor on the device of features")
    dfeat = torch.empty((N, D), dtype=torch.float32, device=dev)
    lib = _L()
    with torch.cuda.device(dev):
        ws = _bytes(lib.gsb_splat_features_workspace_bytes(N, H, W, 0 if recs else P), dev)
        _lib.check(lib.gsb_splat_features_backward(
            H, W, N, P, D, *[_ptr(a) for a in attrs], _ptr(features), recs, _ptr(contrib), _ptr(final_tau), _ptr(ranges),
            _ptr(gsid), _ptr(dl), _ptr(ws), ws.numel(), _ptr(moments), _ptr(dfeat), _stream()), lib)
    return moments, dfeat


# ---------------------------------------------------------------------------------------
# Contribution statistics (extension; DESIGN 3.18): per-Gaussian sums of the blending weights.
def _stats_out(out, N, dev):
    """the accumulators of `splat_stats` / `splat_surfel_stats`: fresh zeros, or the caller's
    (weight_sum[N] f32, weight_max[N] f32, hit_count[N] i64), contiguous, on `dev`"""
    if out is None:
        return (torch.zeros(N, dtype=torch.float32, device=dev), torch.zeros(N, dtype=torch.float32, device=dev),
                torch.zeros(N, dtype=torch.int64, device=dev))
    if not (isinstance(out, (tuple, list)) and len(out) == 3):
        raise ValueError("out must be (weight_sum, weight_max, hit_count)")
    for t, name, dt in zip(out, ("weight_sum", "weight_max", "hit_count"), (torch.float32, torch.float32, torch.int64)):
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dt and tuple(t.shape) == (N,) and
                t.is_contiguous() and t.device == dev):
            raise ValueError("%s must be a contiguous %s [N] tensor on the frame's device" % (name, dt))
    return tuple(out)


def splat_stats(height, width, contrib, patch_range_per_tile, gsid_per_patch, records=None, us=None, cinv2ds=None,
                alphas=None, colors=None, out=None):
    """Contribution statistics of a frame `splat` (or `splat_rgbd`) drew (gsb_splat_stats), with the
    blending weights w = tau alpha' the image composited (the same bits):
        weight_sum[i] += sum_p w_i(p),  weight_max[i] = max(weight_max[i], max_p w_i(p)),
        hit_count[i] += #{p : w_i(p) > 0}.
    contrib, patch_range_per_tile, gsid_per_patch: that frame's outputs.  records, us, cinv2ds,
    alphas, colors: as for `splat_features` (given, attached to gsid_per_patch by `splat`, or
    re-packed); N is taken from records, else from us.  out: (weight_sum[N] f32, weight_max[N] f32,
    hit_count[N] i64) to accumulate into, in place (weight_max must hold values >= 0); None: fresh
    zeros.  -> (weight_sum, weight_max, hit_count)"""
    ref = records if records is not None else us
    if ref is None:
        raise ValueError("give the forward's records, or us, cinv2ds, alphas and colors to find or re-pack them")
    N = ref.shape[0]
    # _feature_frame's checks and record rules, with a [N, 1] stand-in for the features it checks
    H, W, N, _, P, _, contrib, ranges, gsid, recs, attrs = _feature_frame(
        height, width, torch.empty((N, 1), dtype=torch.float32, device=ref.device), contrib, patch_range_per_tile,
        gsid_per_patch, records, us, cinv2ds, alphas, colors)
    dev = contrib.device
    ws_sum, ws_max, hits = _stats_out(out, N, dev)
    lib = _L()
    with torch.cuda.device(dev):
        ws = _bytes(lib.gsb_splat_stats_workspace_bytes(N, H, W, 0 if recs else P), dev)
        _lib.check(lib.gsb_splat_stats(H, W, N, P, *[_ptr(a) for a in attrs], recs, _ptr(contrib), _ptr(ranges),
                                       _ptr(gsid), _ptr(ws), ws.numel(), _ptr(ws_sum), _ptr(ws_max), _ptr(hits),
                                       _stream()), lib)
    return ws_sum, ws_max, hits


# ---------------------------------------------------------------------------------------
# Extensions (not in the reference module): the fused per-Gaussian path, SURVEY 8f row N1.
CAMERA_MODELS = ("pinhole", "ortho", "fisheye", "opencv")
# GSB_CAMERA_*: 3 is not a model (gsplat_b200.h)
_CAMERA_MODEL_ID = {"pinhole": 0, "ortho": 1, "fisheye": 2, "opencv": 4}


class _CameraModel(C.Structure):
    _fields_ = [("model", C.c_int32), ("k", C.c_float * 4)]


def _finite(coeffs, n, what):
    k = tuple(float(x) for x in coeffs)
    if len(k) != n or not all(math.isfinite(x) for x in k):
        raise ValueError("%s must be %d finite numbers %s" % (what[0], n, what[1]))
    return k


def camera_model_args(camera_model="pinhole", radial_coeffs=None, tangential_coeffs=None):
    """Checks a camera model on the host -> (name, the four coefficients of gsb_camera_model.k as
    floats).  camera_model is "pinhole", "ortho", "fisheye" or "opencv"; None coefficients are 0.
    fisheye: radial_coeffs = (k1, k2, k3, k4) of the Kannala-Brandt lens (COLMAP's OPENCV_FISHEYE).
    opencv: radial_coeffs = (k1, k2) and tangential_coeffs = (p1, p2) of COLMAP's OPENCV model
    (RADIAL: p = 0; SIMPLE_RADIAL: k2 = p = 0); k = (k1, k2, p1, p2).  All must be finite."""
    if camera_model not in CAMERA_MODELS:
        raise ValueError("camera_model must be one of %s, got %r" % (CAMERA_MODELS, camera_model))
    if radial_coeffs is not None and camera_model not in ("fisheye", "opencv"):
        raise ValueError("radial_coeffs are for camera_model='fisheye' or 'opencv' only")
    if tangential_coeffs is not None and camera_model != "opencv":
        raise ValueError("tangential_coeffs are for camera_model='opencv' only")
    if camera_model == "opencv":
        k = (0.0, 0.0) if radial_coeffs is None else _finite(radial_coeffs, 2, ("radial_coeffs", "(k1, k2)"))
        p = (0.0, 0.0) if tangential_coeffs is None else _finite(tangential_coeffs, 2,
                                                                ("tangential_coeffs", "(p1, p2)"))
        return camera_model, k + p
    if radial_coeffs is None:
        return camera_model, (0.0, 0.0, 0.0, 0.0)
    return camera_model, _finite(radial_coeffs, 4, ("radial_coeffs", "(k1, k2, k3, k4)"))


def _camera_model_ptr(camera_model, radial_coeffs, tangential_coeffs, focal_x, focal_y):
    """-> None for pinhole (today's entry points), else the gsb_camera_model to pass by pointer"""
    name, k = camera_model_args(camera_model, radial_coeffs, tangential_coeffs)
    if name == "pinhole":
        return None
    if not (float(focal_x) > 0 and float(focal_y) > 0):
        raise ValueError("camera_model=%r needs focal_x, focal_y > 0" % name)
    return C.pointer(_CameraModel(_CAMERA_MODEL_ID[name], (C.c_float * 4)(*k)))


def preprocess(pws, rots, scales, shs, Rcw, tcw, twc, focal_x, focal_y, center_x, center_y, width, height,
               alphas=None, antialiased=False, camera_model="pinhole", radial_coeffs=None, tangential_coeffs=None):
    """project + computeCov3D + computeCov2D + sh2Color + inverseCov2D (calc_J=False) in one
    kernel.  -> [us[N,2], cinv2ds[N,3], colors[N,3], depths[N], areas[N,2] int32], ready for
    `splat`.  With alphas[N] a sixth output: the packed per-Gaussian records [N,12] for
    `splat(..., records=...)`.
    antialiased (alphas required): a seventh output alphas_eff[N] = rho * alphas, the opacity
    scaled by how much the 0.3 px blur spread each Gaussian (gsb_preprocess_forward_aa); the records
    carry it.  Render with alphas_eff; the other outputs are the same bits as without.
    camera_model ("pinhole", "ortho", "fisheye" or "opencv"), radial_coeffs (fisheye's k1..k4,
    opencv's k1, k2) and tangential_coeffs (opencv's p1, p2): the projection
    (gsb_preprocess_forward_model; pinhole runs the calls above; `camera_model_args`).
    width/height feed only pinhole's and opencv's clamp of the EWA Jacobian."""
    cm = _camera_model_ptr(camera_model, radial_coeffs, tangential_coeffs, focal_x, focal_y)
    params, N, k = _gaussian_params(pws, rots, scales, shs, Rcw, tcw, twc)
    pws = params[0]
    if antialiased and alphas is None:
        raise ValueError("antialiased=True needs alphas")
    o = dict(dtype=torch.float32, device=pws.device)
    us = torch.empty((N, 2), **o); cinv = torch.empty((N, 3), **o); col = torch.empty((N, 3), **o)
    depths = torch.empty((N,), **o); areas = torch.empty((N, 2), dtype=torch.int32, device=pws.device)
    records = None
    if alphas is not None:
        alphas = _per_gaussian(alphas, "alphas", N, pws)
        records = torch.empty((N, 12), **o)
    lib = _L()
    with torch.cuda.device(pws.device):
        args = _scene_args(params, N, k, focal_x, focal_y, center_x, center_y, width, height) + (
            _ptr(us), _ptr(cinv), _ptr(col), _ptr(depths), _ptr(areas), _ptr(alphas), _ptr(records))
        alphas_eff = torch.empty((N,), **o) if antialiased else None
        if cm is not None:
            _lib.check(lib.gsb_preprocess_forward_model(*args, _ptr(alphas_eff), cm, _stream()), lib)
        elif antialiased:
            _lib.check(lib.gsb_preprocess_forward_aa(*args, _ptr(alphas_eff), _stream()), lib)
        else:
            _lib.check(lib.gsb_preprocess_forward(*args, _stream()), lib)
        if antialiased:
            return [us, cinv, col, depths, areas, records, alphas_eff]
    return [us, cinv, col, depths, areas] + ([records] if records is not None else [])


def preprocessB(pws, rots, scales, shs, Rcw, tcw, twc, focal_x, focal_y, center_x, center_y, width, height,
                dloss_dus, dloss_dcinv2ds, dloss_dcolors, moments=None, cinv2ds=None, compact=False,
                dloss_ddepths=None, camera_grad=False, pose_only=False, antialiased=False, alphas=None,
                camera_model="pinhole", radial_coeffs=None, tangential_coeffs=None, intrinsics_grad=False):
    """Vector-Jacobian products of the five per-Gaussian stages (== the torch.bmm chain of
    gsmodel.py:72-85).  -> [dloss_dpws[N,3], dloss_dshs[N,3k], dloss_dscales[N,3], dloss_drots[N,4]]
    With moments[N,9] (from `splatB(..., moments_only=True)`) and the forward's cinv2ds[N,3] the
    three dloss_d* arguments are ignored (pass None) and two more outputs follow:
    dloss_dus[N,2], dloss_dalphas[N].
    compact (with moments): dloss_dshs is not produced (None) -- the caller expands it from the
    views' dL/dcolor = moments[:, 6:9] with `sh_grad_expand` -- and the other gradients share one
    flat bucket [dpws | dscales | drots | dalphas] of 11 N floats (one collective sums it).
    dloss_ddepths[N] (from `splatB_rgbd`): dL/dz of the Gaussians' depths; dloss_dpws gains
    dloss_ddepths Rcw[2,:] (0 for culled Gaussians).  None: exactly the colour-only call.
    camera_grad: one more output follows, the camera gradient (dRcw[3,3], dtcw[3], dtwc[3]) --
    views of one 15-float tensor, summed over the Gaussians in a fixed order (gsb_preprocess_backward_pose;
    Rcw, tcw, twc taken as independent inputs).  The per-Gaussian outputs are the same bits as
    without it.  pose_only (with camera_grad): the map is frozen; the per-Gaussian gradients
    (and dloss_dus, dloss_dalphas) are not computed and come back as None.
    antialiased (with moments and the raw alphas[N]): the frame was rendered with
    `preprocess(..., antialiased=True)`'s alphas_eff, so the moment rows' dL/dalpha is dL/dalphas_eff;
    dloss_dalphas = rho * dL/dalphas_eff and the geometry (and camera) gradients gain the term
    through rho (gsb_preprocess_backward_aa).  Combines with compact, dloss_ddepths, camera_grad
    and pose_only.
    camera_model, radial_coeffs, tangential_coeffs: as for `preprocess` (gsb_preprocess_backward_model);
    a model other than pinhole needs the moment rows and combines with everything above.
    intrinsics_grad (with camera_grad and the moment rows; DESIGN 3.23,
    gsb_preprocess_backward_intrinsics): one more output follows the camera gradient, dintrinsics[8] =
    dL/d(focal_x, focal_y, center_x, center_y, k[4]) with k the camera model's coefficients (opencv: k1,
    k2, p1, p2; fisheye: k1..k4; 0 for pinhole and ortho).  The clamp bound, culls and tile rectangles
    are held constant."""
    if intrinsics_grad and (not camera_grad or moments is None):
        raise ValueError("intrinsics_grad=True needs camera_grad=True and the moment rows")
    cm = _camera_model_ptr(camera_model, radial_coeffs, tangential_coeffs, focal_x, focal_y)
    if cm is not None and moments is None:
        raise ValueError("camera_model=%r needs the moment rows" % camera_model)
    if pose_only and not camera_grad:
        raise ValueError("pose_only=True needs camera_grad=True")
    if camera_grad and compact:
        raise ValueError("camera_grad does not combine with compact")
    if antialiased and (moments is None or alphas is None):
        raise ValueError("antialiased=True needs the moment rows and alphas")
    params, N, k = _gaussian_params(pws, rots, scales, shs, Rcw, tcw, twc)
    pws = params[0]
    gu, gc, gcol, moments, cinv2ds = _upstream_grads(N, pws, dloss_dus, dloss_dcinv2ds, dloss_dcolors, moments,
                                                     cinv2ds)
    if antialiased:
        alphas = _per_gaussian(alphas, "alphas", N, pws)
    if dloss_ddepths is not None:
        dloss_ddepths = _per_gaussian(dloss_ddepths, "dloss_ddepths", N, pws)
    o = dict(dtype=torch.float32, device=pws.device)
    # one flat bucket [dshs | drots | dpws | dscales]: a multi-GPU caller can all-reduce the four
    # gradients in place with a single collective (parallel.allreduce_grads); every view starts
    # 16-byte aligned (3k*N and 4*N floats are multiples of 4 elements when N % 4 == 0; the
    # kernels fall back to scalar stores otherwise)
    if pose_only:
        bucket = gsh = gpw = gs = gq = dal = None
    elif compact:
        if moments is None:
            raise ValueError("compact=True needs the moment rows")
        bucket = torch.empty((N * 11,), **o)
        gsh = None
        gpw = bucket[:3 * N].view(N, 3)
        gs = bucket[3 * N:6 * N].view(N, 3)
        gq = bucket[6 * N:10 * N].view(N, 4)
        dal = bucket[10 * N:]
    else:
        bucket = torch.empty((N * (3 * k + 10),), **o)
        gsh = bucket[:N * 3 * k].view(N, 3 * k)
        gq = bucket[N * 3 * k:N * (3 * k + 4)].view(N, 4)
        gpw = bucket[N * (3 * k + 4):N * (3 * k + 7)].view(N, 3)
        gs = bucket[N * (3 * k + 7):].view(N, 3)
        dal = torch.empty((N,), **o) if moments is not None else None
    dus = torch.empty((N, 2), **o) if moments is not None and not pose_only else None
    lib = _L()
    with torch.cuda.device(pws.device):
        args = _scene_args(params, N, k, focal_x, focal_y, center_x, center_y, width, height) + (
            _ptr(gu), _ptr(gc), _ptr(gcol), _ptr(gpw), _ptr(gsh), _ptr(gs), _ptr(gq), _ptr(moments), _ptr(cinv2ds),
            _ptr(dus), _ptr(dal))
        gcam = ws = None
        ws_bytes = 0
        if camera_grad:
            gcam = torch.empty((15,), **o)
            ws_bytes = int(lib.gsb_preprocess_backward_intrinsics_workspace_bytes(N) if intrinsics_grad else
                           lib.gsb_preprocess_backward_pose_workspace_bytes(N))
            ws = torch.empty((max(ws_bytes, 16),), dtype=torch.uint8, device=pws.device)
        if intrinsics_grad:
            gint = torch.empty((8,), **o)
            _lib.check(lib.gsb_preprocess_backward_intrinsics(*args, _ptr(dloss_ddepths),
                                                              _ptr(alphas if antialiased else None), _ptr(gcam),
                                                              _ptr(gint), _ptr(ws), ws_bytes, cm, _stream()), lib)
        elif cm is not None:
            _lib.check(lib.gsb_preprocess_backward_model(*args, _ptr(dloss_ddepths), _ptr(alphas if antialiased else None),
                                                         _ptr(gcam), _ptr(ws), ws_bytes, cm, _stream()), lib)
        elif antialiased:
            _lib.check(lib.gsb_preprocess_backward_aa(*args, _ptr(dloss_ddepths), _ptr(alphas), _ptr(gcam), _ptr(ws),
                                                      ws_bytes, _stream()), lib)
        elif camera_grad:
            _lib.check(lib.gsb_preprocess_backward_pose(*args, _ptr(dloss_ddepths), _ptr(gcam), _ptr(ws), ws_bytes,
                                                        _stream()), lib)
        elif dloss_ddepths is not None:
            _lib.check(lib.gsb_preprocess_backward_rgbd(*args, _ptr(dloss_ddepths), _stream()), lib)
        else:
            _lib.check(lib.gsb_preprocess_backward(*args, _stream()), lib)
    out = [gpw, gsh, gs, gq] + ([dus, dal] if moments is not None else [])
    if camera_grad:
        out.append((gcam[:9].view(3, 3), gcam[9:12], gcam[12:15]))
    if intrinsics_grad:
        out.append(gint)
    return out


# ---------------------------------------------------------------------------------------
# Mip-Splatting's 3D smoothing filter (gsb_filter3d*): a per-Gaussian lower bound on the size,
# from the sampling rate of the training views.  scales / alphas are the activated values.
FILTER3D_CHUNK = 64   # cameras the filter kernel stages in shared memory at once (GSB_FILTER3D_CHUNK)
CAMERA_ROW = 20       # Rcw (row-major 9), tcw (3), fx, fy, cx, cy, W, H, 2 unused


def camera_table(cams, device=None):
    """Packs training cameras -- any objects with the reference Camera's fields width, height, fx,
    fy, cx, cy, Rcw[3,3], tcw[3] (gsplat/gausplat_dataset.py Camera, gsfunction.Camera) -- into the
    [C, 20] float32 device table `filter3d` reads.  W, H > 0 and finite intrinsics with fx > 0 are
    checked here, on the host.  device: where the table goes (default: that of the first
    camera's Rcw when it is a CUDA tensor, else the current CUDA device)."""
    cams = list(cams)
    rows = torch.zeros((len(cams), CAMERA_ROW), dtype=torch.float64)
    for k, c in enumerate(cams):
        if getattr(c, "camera_model", "pinhole") != "pinhole":
            # the visibility test and the d / f sampling rate are pinhole formulas
            raise ValueError("camera %d: the 3D filter is computed from pinhole cameras only, got camera_model=%r"
                             % (k, c.camera_model))
        w, h = float(c.width), float(c.height)
        intr = [float(c.fx), float(c.fy), float(c.cx), float(c.cy)]
        if not (w > 0 and h > 0):
            raise ValueError("camera %d: width and height must be positive" % k)
        if not all(math.isfinite(x) for x in intr) or intr[0] <= 0:
            raise ValueError("camera %d: fx, fy, cx, cy must be finite and fx > 0" % k)
        R = torch.as_tensor(c.Rcw).detach().reshape(-1).to("cpu", torch.float64)
        t = torch.as_tensor(c.tcw).detach().reshape(-1).to("cpu", torch.float64)
        if R.numel() != 9 or t.numel() != 3:
            raise ValueError("camera %d: Rcw must have 9 and tcw 3 elements" % k)
        rows[k, :9], rows[k, 9:12] = R, t
        rows[k, 12:18] = torch.tensor(intr + [w, h], dtype=torch.float64)
    if device is None:
        R0 = cams[0].Rcw if cams else None
        device = R0.device if isinstance(R0, torch.Tensor) and R0.is_cuda else torch.device("cuda")
    return rows.to(torch.float32).to(device)


def filter3d(pws, cams_or_table, variance=0.2):
    """The 3D filter of every Gaussian from the training cameras (gsb_filter3d): camera k sees
    Gaussian i when its camera-frame depth z >= 0.2 and its projected mean lies within 15 % of the
    frame on every side; d_i = the smallest such z (the largest d of the seen Gaussians when no
    camera sees i), and filter3d_i = sqrt(variance) d_i / max_k fx_k (the largest positive fx; a
    table given as a tensor is not checked on the host).  All 0 when nothing is seen or no camera
    has fx > 0.
    cams_or_table: camera objects (`camera_table`) or such a [C, 20] table.  -> filter3d[N]"""
    pws = _chk(pws, "pws", last=3, ndim=2)
    if isinstance(cams_or_table, torch.Tensor):
        table = _chk(cams_or_table, "camera table", last=CAMERA_ROW, ndim=2)
    else:
        table = camera_table(cams_or_table, device=pws.device)
    _same_device(pws, table)
    variance = float(variance)
    if not (math.isfinite(variance) and variance >= 0):
        raise ValueError("variance must be finite and >= 0")
    N, Cn = pws.shape[0], table.shape[0]
    out = torch.empty((N,), dtype=torch.float32, device=pws.device)
    lib = _L()
    nbytes = int(lib.gsb_filter3d_workspace_bytes(N, Cn))
    ws = _bytes(max(nbytes, 16), pws.device)
    with torch.cuda.device(pws.device):
        _lib.check(lib.gsb_filter3d(N, _ptr(pws), Cn, _ptr(table), variance, _ptr(out), _ptr(ws), nbytes, _stream()),
                   lib)
    return out


def _filter3d_rows(scales, alphas, filter3d):
    scales = _chk(scales, "scales", last=3, ndim=2); alphas = _chk(alphas, "alphas")
    filter3d = _chk(filter3d, "filter3d")
    _same_device(scales, alphas, filter3d)
    N = scales.shape[0]
    if alphas.numel() != N or filter3d.numel() != N:
        raise ValueError("scales[N,3], alphas[N] and filter3d[N] disagree on N")
    return scales, alphas, filter3d, N


def filter3d_apply(scales, alphas, filter3d):
    """(scales[N,3], alphas) -> (scales_f, alphas_f) (gsb_filter3d_apply): s'_j = sqrt(s_j^2 + f^2)
    and alpha' = alpha prod_j s_j / s'_j, which keeps each Gaussian's mass; f == 0 copies exactly.
    alphas_f has the shape of alphas.  Render with these; the filter itself is not differentiated."""
    shape = alphas.shape if isinstance(alphas, torch.Tensor) else None
    scales, alphas, filter3d, N = _filter3d_rows(scales, alphas, filter3d)
    sf = torch.empty_like(scales); af = torch.empty(shape, dtype=torch.float32, device=scales.device)
    lib = _L()
    with torch.cuda.device(scales.device):
        _lib.check(lib.gsb_filter3d_apply(N, _ptr(scales), _ptr(alphas), _ptr(filter3d), _ptr(sf), _ptr(af),
                                          _stream()), lib)
    return sf, af


def filter3d_backward(scales, alphas, filter3d, dloss_dscales_f, dloss_dalphas_f, inplace=False):
    """Backward of `filter3d_apply` (gsb_filter3d_backward): dL/ds' [N,3] and dL/dalpha' -> (dL/ds,
    dL/dalpha) of the unfiltered scales and alphas.  inplace: written over the two gradient inputs
    (which must then be contiguous float32 CUDA tensors) and those are returned."""
    scales, alphas, filter3d, N = _filter3d_rows(scales, alphas, filter3d)
    if inplace and not (isinstance(dloss_dscales_f, torch.Tensor) and dloss_dscales_f.is_contiguous() and
                        isinstance(dloss_dalphas_f, torch.Tensor) and dloss_dalphas_f.is_contiguous()):
        raise ValueError("inplace=True needs contiguous gradient tensors")
    gs = _chk(dloss_dscales_f, "dloss_dscales_f", last=3, ndim=2)
    ga_shape = dloss_dalphas_f.shape if isinstance(dloss_dalphas_f, torch.Tensor) else None
    ga = _chk(dloss_dalphas_f, "dloss_dalphas_f")
    _same_device(scales, gs, ga)
    if gs.shape[0] != N or ga.numel() != N:
        raise ValueError("dloss_dscales_f[N,3] and dloss_dalphas_f[N] disagree with scales on N")
    if inplace:
        ds, da = gs, ga
    else:
        ds = torch.empty_like(gs); da = torch.empty(ga_shape, dtype=torch.float32, device=gs.device)
    lib = _L()
    with torch.cuda.device(scales.device):
        _lib.check(lib.gsb_filter3d_backward(N, _ptr(scales), _ptr(alphas), _ptr(filter3d), _ptr(gs), _ptr(ga),
                                             _ptr(ds), _ptr(da), _stream()), lib)
    return ds, da


def sh_grad_expand(pws, twcs, dloss_dcolors, sh_dim3, out=None):
    """dloss_dshs[N, 3k] = sum over the V views of Y(dir_v) (x) dloss_dcolors[v]  (gsb_sh_grad_expand;
    colour is linear in sh, kernel.cu:735-774).  pws[N,3], twcs[V,3] (camera centres),
    dloss_dcolors[V,N,3]."""
    pws = _chk(pws, "pws", last=3, ndim=2); twcs = _chk(twcs, "twcs", last=3, ndim=2)
    g = _chk(dloss_dcolors, "dloss_dcolors", last=3, ndim=3)
    _same_device(pws, twcs, g)
    N, V, k = pws.shape[0], twcs.shape[0], int(sh_dim3)
    if g.shape[0] != V or g.shape[1] != N or k not in (1, 4, 9, 16):
        raise ValueError("sh_grad_expand: need twcs[V,3], dloss_dcolors[V,N,3], sh_dim3 in {1,4,9,16}")
    if out is None:
        out = torch.empty((N, 3 * k), dtype=torch.float32, device=pws.device)
    else:  # the kernel writes N * 3k floats through out's data pointer
        if not isinstance(out, torch.Tensor) or out.dtype != torch.float32:
            raise TypeError("out must be a float32 torch.Tensor")
        if out.device != pws.device:
            raise ValueError("out must be on the device of pws")
        if tuple(out.shape) != (N, 3 * k) or not out.is_contiguous():
            raise ValueError("out must be a contiguous (%d, %d) tensor, got shape %s" % (N, 3 * k, tuple(out.shape)))
    lib = _L()
    with torch.cuda.device(pws.device):
        _lib.check(lib.gsb_sh_grad_expand(N, k, V, _ptr(pws), _ptr(twcs), _ptr(g), _ptr(out), _stream()), lib)
    return out


# ---------------------------------------------------------------------------------------
# 2D Gaussian Splatting (extension; DESIGN 3.15): surfels drawn by ray-splat intersection.
SURFEL_RECORD = 20  # floats per surfel record (80 bytes)
SURFEL_ROW = 18     # floats per gradient row: dM (9), dalpha, dcolour (3), dn (3), ddelta (2)


def surfel_preprocess(pws, rots, scales, shs, alphas, Rcw, tcw, twc, focal_x, focal_y, center_x, center_y, width,
                      height):
    """The per-surfel forward (gsb_surfel_preprocess_forward): scales[:, 0] and scales[:, 1] are the
    disk's axes (column 2 is not read), rots its (normalised here) quaternion, pinhole camera.
    -> (us[N,2], depths[N] (-1 = culled), areas[N,2] i32, colors[N,3], records[N,20])"""
    params, N, k = _gaussian_params(pws, rots, scales, shs, Rcw, tcw, twc)
    alphas = _per_gaussian(alphas, "alphas", N, params[0])
    o = dict(dtype=torch.float32, device=params[0].device)
    us = torch.empty((N, 2), **o); depths = torch.empty((N,), **o); colors = torch.empty((N, 3), **o)
    areas = torch.empty((N, 2), dtype=torch.int32, device=params[0].device)
    records = torch.empty((N, SURFEL_RECORD), **o)
    lib = _L()
    with torch.cuda.device(params[0].device):
        _lib.check(lib.gsb_surfel_preprocess_forward(
            *_scene_args(params, N, k, focal_x, focal_y, center_x, center_y, width, height), _ptr(alphas), _ptr(us),
            _ptr(depths), _ptr(areas), _ptr(colors), _ptr(records), _stream()), lib)
    return us, depths, areas, colors, records


def surfel_preprocessB(pws, rots, scales, shs, Rcw, tcw, twc, focal_x, focal_y, center_x, center_y, width, height,
                       rows):
    """The per-surfel backward (gsb_surfel_preprocess_backward) from splatB_surfel's rows[N,18].
    -> (dpws[N,3], dshs[N,3k], dalphas[N], dscales[N,3] (column 2: 0), drots[N,4], dus[N,2])"""
    params, N, k = _gaussian_params(pws, rots, scales, shs, Rcw, tcw, twc)
    rows = _chk(rows, "rows", last=SURFEL_ROW, ndim=2)
    _same_device(params[0], rows)
    if rows.shape[0] != N:
        raise ValueError("rows must be [N, %d]" % SURFEL_ROW)
    o = dict(dtype=torch.float32, device=params[0].device)
    out = (torch.empty((N, 3), **o), torch.empty((N, 3 * k), **o), torch.empty((N,), **o), torch.empty((N, 3), **o),
           torch.empty((N, 4), **o), torch.empty((N, 2), **o))
    lib = _L()
    with torch.cuda.device(params[0].device):
        _lib.check(lib.gsb_surfel_preprocess_backward(
            *_scene_args(params, N, k, focal_x, focal_y, center_x, center_y, width, height), _ptr(rows),
            *[_ptr(t) for t in out], _stream()), lib)
    return out


def splat_surfel(height, width, us, depths, areas, records, capacity=False):
    """Bins the surfels (us, areas, depths: the binning of `splat`, which MUTATES depths / areas of
    surfels that touch no tile) and draws them.  -> [image[3,H,W], contrib[H,W] i32,
    final_tau[H,W], patch_range_per_tile[T,2] i32, gsid_per_patch[P] i32, depth[H,W], alpha[H,W],
    normal[3,H,W]] with depth = sum w z(p) (the camera-frame depth of each ray-splat hit, not
    normalised), alpha = sum w, normal = sum w n (camera frame), w = tau alpha'.
    capacity: as for `splat` (sort sized from the previous frame of this shape; an outgrown frame
    is redone the exact way)."""
    H, W = int(height), int(width)
    if H <= 0 or W <= 0:
        raise ValueError("height and width must be positive")
    us = _chk(us, "us", last=2, ndim=2); depths = _chk(depths, "depths")
    areas = _chk(areas, "areas", dtype=torch.int32, last=2, ndim=2)
    records = _chk(records, "records", last=SURFEL_RECORD, ndim=2)
    _same_device(us, depths, areas, records)
    N = us.shape[0]
    if not (depths.numel() == N and areas.shape[0] == N and records.shape[0] == N):
        raise ValueError("splat_surfel inputs disagree on N")
    dev, lib = us.device, _L()
    with torch.cuda.device(dev):
        _, _, out = _frame(H, W, us, depths, areas, [(H, W), (H, W), (3, H, W)], lib.gsb_splat_surfel_workspace_bytes,
                           (lib.gsb_splat_surfel_forward, [_ptr(us), _ptr(depths), _ptr(areas), _ptr(records)]),
                           (lib.gsb_splat_surfel_render, [_ptr(us), _ptr(depths), _ptr(records)]), capacity,
                           ("surfel", dev.index, H, W, N))
    return out


def splatB_surfel(height, width, records, contrib, final_tau, patch_range_per_tile, gsid_per_patch,
                  dloss_dimage=None, dloss_ddepth=None, dloss_dalpha=None, dloss_dnormal=None):
    """Backward of `splat_surfel` from the planes' upstream gradients ([3,H,W], [H,W], [H,W],
    [3,H,W]; None = zero and not read; all None: no rasterizer pass, zero rows).
    -> rows[N,18] = [dL/dM (9), dL/dalpha, dL/dcolour (3), dL/dn (3), dL/ddelta (2)] per surfel,
    for `surfel_preprocessB`"""
    H, W = int(height), int(width)
    records = _chk(records, "records", last=SURFEL_RECORD, ndim=2)
    contrib = _chk(contrib, "contrib", dtype=torch.int32); final_tau = _chk(final_tau, "final_tau")
    ranges = _chk(patch_range_per_tile, "patch_range_per_tile", dtype=torch.int32, last=2)
    gsid = _chk(gsid_per_patch, "gsid_per_patch", dtype=torch.int32)
    _same_device(records, contrib, final_tau, ranges, gsid)
    _check_drawn(H, W, ranges, ((contrib, 1), (final_tau, 1)), "contrib / final_tau do not match height x width")
    planes = []
    for name, t, n in (("dloss_dimage", dloss_dimage, 3), ("dloss_ddepth", dloss_ddepth, 1),
                       ("dloss_dalpha", dloss_dalpha, 1), ("dloss_dnormal", dloss_dnormal, 3)):
        if t is not None:
            t = _chk(t, name)
            _same_device(records, t)
            if t.numel() != n * H * W:
                raise ValueError("%s does not match height x width" % name)
        planes.append(t)
    N, P, dev, lib = records.shape[0], gsid.numel(), records.device, _L()
    rows = torch.empty((N, SURFEL_ROW), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        ws = _bytes(lib.gsb_splat_surfel_workspace_bytes(N, H, W, 0), dev)
        _lib.check(lib.gsb_splat_surfel_backward(H, W, N, P, _ptr(records), _ptr(contrib), _ptr(final_tau),
                                                 _ptr(ranges), _ptr(gsid), *[_ptr(t) for t in planes], _ptr(ws),
                                                 ws.numel(), _ptr(rows), _stream()), lib)
    return rows


def splat_surfel_stats(height, width, records, contrib, patch_range_per_tile, gsid_per_patch, out=None):
    """`splat_stats` for a frame `splat_surfel` / `splat_surfel_geometry` drew from records[N,20]
    (gsb_splat_stats_2dgs): the same three statistics with the surfel frame's weights (its bits).
    out: as for `splat_stats`.  -> (weight_sum, weight_max, hit_count)"""
    H, W = int(height), int(width)
    if H <= 0 or W <= 0:
        raise ValueError("height and width must be positive")
    records = _chk(records, "records", last=SURFEL_RECORD, ndim=2)
    contrib = _chk(contrib, "contrib", dtype=torch.int32)
    ranges = _chk(patch_range_per_tile, "patch_range_per_tile", dtype=torch.int32, last=2)
    gsid = _chk(gsid_per_patch, "gsid_per_patch", dtype=torch.int32)
    _same_device(records, contrib, ranges, gsid)
    _check_drawn(H, W, ranges, ((contrib, 1),), "contrib does not match height x width")
    N, P, dev, lib = records.shape[0], gsid.numel(), records.device, _L()
    ws_sum, ws_max, hits = _stats_out(out, N, dev)
    with torch.cuda.device(dev):
        _lib.check(lib.gsb_splat_stats_2dgs(H, W, N, P, _ptr(records), _ptr(contrib), _ptr(ranges), _ptr(gsid),
                                              _ptr(ws_sum), _ptr(ws_max), _ptr(hits), _stream()), lib)
    return ws_sum, ws_max, hits


# 2DGS geometry terms (extension; DESIGN 3.16): depth distortion and median depth of the surfel frame.
def _near_far(near, far):
    """near / far of the geometry planes: plain numbers (not tensors), finite, 0 < near < far"""
    if not all(isinstance(x, numbers.Real) and not isinstance(x, bool) for x in (near, far)):
        raise ValueError("near and far must be numbers (there is no filter3d or us_abs argument)")
    near, far = float(near), float(far)
    if not (math.isfinite(near) and math.isfinite(far) and 0.0 < near < far):
        raise ValueError("near and far must be finite with 0 < near < far")
    return near, far


def splat_surfel_geometry(height, width, us, depths, areas, records, near=0.2, far=100.0, capacity=False):
    """`splat_surfel` (the same binning, the same eight outputs bit for bit) with 2DGS's geometry
    planes.  -> splat_surfel's eight outputs + [distortion[H,W], median_depth[H,W], moments[2,H,W],
    median_contrib[H,W] i32], per pixel over the contributing surfels in compositing order
    (w = tau alpha', z the hit depth, m(z) = far / (far - near) (1 - near / max(z, near))):
        distortion = sum_{j<i} w_i w_j (m_i - m_j)^2,   moments = (sum w m, sum w m^2),
        median_depth = z of the last surfel whose incoming tau > 0.5 (0 where none contributes),
    median_contrib its patch index in the tile + 1 (as contrib).  moments and median_contrib are
    what `splatB_surfel_geometry` reads back."""
    H, W = int(height), int(width)
    if H <= 0 or W <= 0:
        raise ValueError("height and width must be positive")
    near, far = _near_far(near, far)
    us = _chk(us, "us", last=2, ndim=2); depths = _chk(depths, "depths")
    areas = _chk(areas, "areas", dtype=torch.int32, last=2, ndim=2)
    records = _chk(records, "records", last=SURFEL_RECORD, ndim=2)
    _same_device(us, depths, areas, records)
    N = us.shape[0]
    if not (depths.numel() == N and areas.shape[0] == N and records.shape[0] == N):
        raise ValueError("splat_surfel_geometry inputs disagree on N")
    dev, lib = us.device, _L()
    planes = [(H, W), (H, W), (3, H, W), (H, W), (2, H, W), (H, W), ((H, W), torch.int32)]
    nf = [C.c_float(near), C.c_float(far)]
    with torch.cuda.device(dev):
        _, _, out = _frame(H, W, us, depths, areas, planes, lib.gsb_splat_surfel_workspace_bytes,
                           (lib.gsb_splat_2dgs_forward, [_ptr(us), _ptr(depths), _ptr(areas), _ptr(records)] + nf),
                           (lib.gsb_splat_2dgs_render, [_ptr(us), _ptr(depths), _ptr(records)] + nf), capacity,
                           ("surfel", dev.index, H, W, N))
    distortion, moments, median_depth, median_contrib = out[8:]
    return out[:8] + [distortion, median_depth, moments, median_contrib]


def splatB_surfel_geometry(height, width, records, contrib, final_tau, patch_range_per_tile, gsid_per_patch,
                           alpha, moments, median_contrib, dloss_dimage=None, dloss_ddepth=None, dloss_dalpha=None,
                           dloss_dnormal=None, dloss_ddistortion=None, dloss_dmedian=None, near=0.2, far=100.0):
    """Backward of `splat_surfel_geometry`: `splatB_surfel`'s upstream planes plus
    dloss_ddistortion[H,W] and dloss_dmedian[H,W] (None = zero and not read); alpha, moments and
    median_contrib are the forward's planes.  -> rows[N,18] as `splatB_surfel`.  With both geometry
    gradients None this is `splatB_surfel` (same kernel, same rows)."""
    if dloss_ddistortion is None and dloss_dmedian is None:
        return splatB_surfel(height, width, records, contrib, final_tau, patch_range_per_tile, gsid_per_patch,
                             dloss_dimage, dloss_ddepth, dloss_dalpha, dloss_dnormal)
    H, W = int(height), int(width)
    near, far = _near_far(near, far)
    records = _chk(records, "records", last=SURFEL_RECORD, ndim=2)
    contrib = _chk(contrib, "contrib", dtype=torch.int32); final_tau = _chk(final_tau, "final_tau")
    ranges = _chk(patch_range_per_tile, "patch_range_per_tile", dtype=torch.int32, last=2)
    gsid = _chk(gsid_per_patch, "gsid_per_patch", dtype=torch.int32)
    alpha = _chk(alpha, "alpha"); moments = _chk(moments, "moments")
    median_contrib = _chk(median_contrib, "median_contrib", dtype=torch.int32)
    _same_device(records, contrib, final_tau, ranges, gsid, alpha, moments, median_contrib)
    _check_drawn(H, W, ranges, ((contrib, 1), (final_tau, 1), (alpha, 1), (moments, 2), (median_contrib, 1)),
                 "contrib / final_tau / alpha / moments / median_contrib do not match height x width")
    planes = []
    for name, t, n in (("dloss_dimage", dloss_dimage, 3), ("dloss_ddepth", dloss_ddepth, 1),
                       ("dloss_dalpha", dloss_dalpha, 1), ("dloss_dnormal", dloss_dnormal, 3),
                       ("dloss_ddistortion", dloss_ddistortion, 1), ("dloss_dmedian", dloss_dmedian, 1)):
        if t is not None:
            t = _chk(t, name)
            _same_device(records, t)
            if t.numel() != n * H * W:
                raise ValueError("%s does not match height x width" % name)
        planes.append(t)
    N, P, dev, lib = records.shape[0], gsid.numel(), records.device, _L()
    rows = torch.empty((N, SURFEL_ROW), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        ws = _bytes(lib.gsb_splat_surfel_workspace_bytes(N, H, W, 0), dev)
        _lib.check(lib.gsb_splat_2dgs_backward(H, W, N, P, _ptr(records), _ptr(contrib), _ptr(final_tau),
                                               _ptr(ranges), _ptr(gsid), *[_ptr(t) for t in planes[:4]], _ptr(ws),
                                               ws.numel(), _ptr(rows), near, far, _ptr(alpha), _ptr(moments),
                                               _ptr(median_contrib), *[_ptr(t) for t in planes[4:]], _stream()), lib)
    return rows


# ---------------------------------------------------------------------------------------
# Batched 2D Gaussian Splatting (extension; DESIGN 3.25): the surfel path for C pinhole cameras of one
# image size in one call, laid out as the batched rendering above (record c N + n = surfel n seen by
# camera c; per-record outputs [C, N, ...], per-pixel ones [C, ..., H, W]).  Frame c is the single
# frame of camera c, bit for bit.
def _surfel_batch_cams(cams, device):
    bc = _batch_cams(cams, device)
    if bc.camera_model != "pinhole" or bc.antialiased:
        raise ValueError("surfel batches take pinhole cameras without antialiasing, got camera_model=%r, "
                         "antialiased=%s" % (bc.camera_model, bc.antialiased))
    return bc


def surfel_preprocess_batch(pws, rots, scales, shs, alphas, cams):
    """`surfel_preprocess` for C cameras at once (gsb_2dgs_batch_preprocess_forward).  cams: a list of
    pinhole `gsfunction.Camera` of one size (or a `BatchCameras`).  -> (us[C,N,2], depths[C,N],
    areas[C,N,2] i32, colors[C,N,3], records[C N, 20]); camera c's rows are the bits
    `surfel_preprocess` gives for camera c alone."""
    (pws, rots, scales, shs), N, k = _gaussian_map(pws, rots, scales, shs)
    bc = _surfel_batch_cams(cams, pws.device)
    alphas = _per_gaussian(alphas, "alphas", N, pws)
    Cn = bc.C
    o = dict(dtype=torch.float32, device=pws.device)
    us = torch.empty((Cn, N, 2), **o); depths = torch.empty((Cn, N), **o); colors = torch.empty((Cn, N, 3), **o)
    areas = torch.empty((Cn, N, 2), dtype=torch.int32, device=pws.device)
    records = torch.empty((Cn * N, SURFEL_RECORD), **o)
    lib = _L()
    with torch.cuda.device(pws.device):
        _lib.check(lib.gsb_2dgs_batch_preprocess_forward(
            Cn, N, k, _ptr(pws), _ptr(rots), _ptr(scales), _ptr(shs), *bc.args(), _ptr(alphas), _ptr(us),
            _ptr(depths), _ptr(areas), _ptr(colors), _ptr(records), _stream()), lib)
    return us, depths, areas, colors, records


def surfel_preprocessB_batch(pws, rots, scales, shs, cams, rows):
    """Backward of `surfel_preprocess_batch` from the rows [C N, 18] of `splatB_surfel_batch` /
    `splatB_surfel_geometry_batch` (gsb_2dgs_batch_preprocess_backward): the C cameras' contributions
    summed in fp32 registers in camera order.  -> (dpws[N,3], dshs[N,3k], dalphas[N], dscales[N,3]
    (column 2: 0), drots[N,4], dus[C,N,2] (per camera))"""
    (pws, rots, scales, shs), N, k = _gaussian_map(pws, rots, scales, shs)
    bc = _surfel_batch_cams(cams, pws.device)
    Cn = bc.C
    rows = _chk(rows, "rows", last=SURFEL_ROW, ndim=2)
    _same_device(pws, rows)
    if rows.shape[0] != Cn * N:
        raise ValueError("rows must be [C N, %d]" % SURFEL_ROW)
    o = dict(dtype=torch.float32, device=pws.device)
    out = (torch.empty((N, 3), **o), torch.empty((N, 3 * k), **o), torch.empty((N,), **o), torch.empty((N, 3), **o),
           torch.empty((N, 4), **o), torch.empty((Cn, N, 2), **o))
    lib = _L()
    with torch.cuda.device(pws.device):
        _lib.check(lib.gsb_2dgs_batch_preprocess_backward(
            Cn, N, k, _ptr(pws), _ptr(rots), _ptr(scales), _ptr(shs), *bc.args(), _ptr(rows),
            *[_ptr(t) for t in out], _stream()), lib)
    return out


def _surfel_batch_inputs(us, depths, areas, records):
    """the [C, N, ...] inputs of a batched surfel frame, checked -> (C, N, us, depths, areas, records)"""
    us = _chk(us, "us", last=2, ndim=3); depths = _chk(depths, "depths")
    areas = _chk(areas, "areas", dtype=torch.int32, last=2, ndim=3)
    records = _chk(records, "records", last=SURFEL_RECORD, ndim=2)
    _same_device(us, depths, areas, records)
    Cn, N = us.shape[0], us.shape[1]
    if not (depths.numel() == Cn * N and tuple(areas.shape[:2]) == (Cn, N) and records.shape[0] == Cn * N):
        raise ValueError("batched surfel frame inputs disagree on C, N")
    return Cn, N, us, depths, areas, records


def splat_surfel_batch(height, width, us, depths, areas, records, capacity=False):
    """`splat_surfel` of C frames at once, binned and drawn as one tall frame (gsb_2dgs_batch_render /
    _forward).  Inputs are `surfel_preprocess_batch`'s; MUTATES depths / areas of records that touch
    no tile.  -> [image[C,3,H,W], contrib[C,H,W] i32, final_tau[C,H,W], patch_range_per_tile[C T,2]
    i32, gsid_per_patch[P] i32 (record ids c N + n), depth[C,H,W], alpha[C,H,W], normal[C,3,H,W]].
    capacity: as for `splat_surfel`."""
    H, W = int(height), int(width)
    if H <= 0 or W <= 0:
        raise ValueError("height and width must be positive")
    Cn, N, us, depths, areas, records = _surfel_batch_inputs(us, depths, areas, records)
    dev, lib = us.device, _L()
    with torch.cuda.device(dev):
        _, _, out = _frame(H, W, us, depths, areas, [(H, W), (H, W), (3, H, W)], lib.gsb_2dgs_batch_workspace_bytes,
                           (lib.gsb_2dgs_batch_forward, [_ptr(us), _ptr(depths), _ptr(areas), _ptr(records)]),
                           (lib.gsb_2dgs_batch_render, [_ptr(us), _ptr(depths), _ptr(records)]), capacity,
                           ("surfel_batch", dev.index, Cn, H, W, N), frames=Cn)
    return out


def splat_surfel_geometry_batch(height, width, us, depths, areas, records, near=0.2, far=100.0, capacity=False):
    """`splat_surfel_geometry` of C frames at once (gsb_2dgs_batch_render_geometry / _forward_geometry):
    `splat_surfel_batch`'s eight outputs + [distortion[C,H,W], median_depth[C,H,W], moments[C,2,H,W],
    median_contrib[C,H,W] i32]."""
    H, W = int(height), int(width)
    if H <= 0 or W <= 0:
        raise ValueError("height and width must be positive")
    near, far = _near_far(near, far)
    Cn, N, us, depths, areas, records = _surfel_batch_inputs(us, depths, areas, records)
    dev, lib = us.device, _L()
    planes = [(H, W), (H, W), (3, H, W), (H, W), (2, H, W), (H, W), ((H, W), torch.int32)]
    nf = [C.c_float(near), C.c_float(far)]
    with torch.cuda.device(dev):
        _, _, out = _frame(H, W, us, depths, areas, planes, lib.gsb_2dgs_batch_workspace_bytes,
                           (lib.gsb_2dgs_batch_forward_geometry, [_ptr(us), _ptr(depths), _ptr(areas), _ptr(records)]
                            + nf),
                           (lib.gsb_2dgs_batch_render_geometry, [_ptr(us), _ptr(depths), _ptr(records)] + nf), capacity,
                           ("surfel_batch", dev.index, Cn, H, W, N), frames=Cn)
    distortion, moments, median_depth, median_contrib = out[8:]
    return out[:8] + [distortion, median_depth, moments, median_contrib]


def _surfel_batch_drawn(H, W, records, contrib, final_tau, patch_range_per_tile, gsid_per_patch, planes):
    """the drawn batch frame of a backward, checked: C from contrib [C,H,W]; planes: (name, tensor or
    None, channels) of [C, channels, H, W] -> (C, N, records, contrib, final_tau, ranges, gsid, tensors)"""
    records = _chk(records, "records", last=SURFEL_RECORD, ndim=2)
    contrib = _chk(contrib, "contrib", dtype=torch.int32, ndim=3); final_tau = _chk(final_tau, "final_tau")
    ranges = _chk(patch_range_per_tile, "patch_range_per_tile", dtype=torch.int32, last=2)
    gsid = _chk(gsid_per_patch, "gsid_per_patch", dtype=torch.int32)
    _same_device(records, contrib, final_tau, ranges, gsid)
    Cn = contrib.shape[0]
    _check_drawn(H, W, ranges, ((contrib, 1), (final_tau, 1)), "contrib / final_tau do not match C x height x width",
                 frames=Cn)
    if records.shape[0] % max(Cn, 1) != 0:
        raise ValueError("records must be [C N, %d]" % SURFEL_RECORD)
    out = []
    for name, t, n in planes:
        if t is not None:
            t = _chk(t, name)
            _same_device(records, t)
            if t.numel() != Cn * n * H * W:
                raise ValueError("%s does not match C x height x width" % name)
        out.append(t)
    return Cn, records.shape[0] // max(Cn, 1), records, contrib, final_tau, ranges, gsid, out


def splatB_surfel_batch(height, width, records, contrib, final_tau, patch_range_per_tile, gsid_per_patch,
                        dloss_dimage=None, dloss_ddepth=None, dloss_dalpha=None, dloss_dnormal=None):
    """Backward of `splat_surfel_batch` (gsb_2dgs_batch_backward) from the planes' upstream gradients
    ([C,3,H,W], [C,H,W], [C,H,W], [C,3,H,W]; None = zero and not read; all None: no rasterizer pass,
    zero rows).  -> rows[C N, 18] for `surfel_preprocessB_batch`"""
    H, W = int(height), int(width)
    Cn, N, records, contrib, final_tau, ranges, gsid, planes = _surfel_batch_drawn(
        H, W, records, contrib, final_tau, patch_range_per_tile, gsid_per_patch,
        (("dloss_dimage", dloss_dimage, 3), ("dloss_ddepth", dloss_ddepth, 1), ("dloss_dalpha", dloss_dalpha, 1),
         ("dloss_dnormal", dloss_dnormal, 3)))
    P, dev, lib = gsid.numel(), records.device, _L()
    rows = torch.empty((Cn * N, SURFEL_ROW), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        ws = _bytes(lib.gsb_2dgs_batch_workspace_bytes(Cn, N, H, W, 0), dev)
        _lib.check(lib.gsb_2dgs_batch_backward(Cn, H, W, N, P, _ptr(records), _ptr(contrib), _ptr(final_tau),
                                               _ptr(ranges), _ptr(gsid), *[_ptr(t) for t in planes], _ptr(ws),
                                               ws.numel(), _ptr(rows), _stream()), lib)
    return rows


def splatB_surfel_geometry_batch(height, width, records, contrib, final_tau, patch_range_per_tile, gsid_per_patch,
                                 alpha, moments, median_contrib, dloss_dimage=None, dloss_ddepth=None,
                                 dloss_dalpha=None, dloss_dnormal=None, dloss_ddistortion=None, dloss_dmedian=None,
                                 near=0.2, far=100.0):
    """Backward of `splat_surfel_geometry_batch` (gsb_2dgs_batch_backward_geometry): `splatB_surfel_batch`'s
    upstream planes plus dloss_ddistortion[C,H,W] and dloss_dmedian[C,H,W]; alpha, moments and
    median_contrib are the forward's planes.  -> rows[C N, 18].  With both geometry gradients None
    this is `splatB_surfel_batch` (same kernel, same rows)."""
    if dloss_ddistortion is None and dloss_dmedian is None:
        return splatB_surfel_batch(height, width, records, contrib, final_tau, patch_range_per_tile, gsid_per_patch,
                                   dloss_dimage, dloss_ddepth, dloss_dalpha, dloss_dnormal)
    H, W = int(height), int(width)
    near, far = _near_far(near, far)
    Cn, N, records, contrib, final_tau, ranges, gsid, planes = _surfel_batch_drawn(
        H, W, records, contrib, final_tau, patch_range_per_tile, gsid_per_patch,
        (("dloss_dimage", dloss_dimage, 3), ("dloss_ddepth", dloss_ddepth, 1), ("dloss_dalpha", dloss_dalpha, 1),
         ("dloss_dnormal", dloss_dnormal, 3), ("dloss_ddistortion", dloss_ddistortion, 1),
         ("dloss_dmedian", dloss_dmedian, 1), ("alpha", alpha, 1), ("moments", moments, 2)))
    alpha, moments = planes[6:]
    median_contrib = _chk(median_contrib, "median_contrib", dtype=torch.int32)
    _same_device(records, median_contrib)
    if median_contrib.numel() != Cn * H * W:
        raise ValueError("median_contrib does not match C x height x width")
    P, dev, lib = gsid.numel(), records.device, _L()
    rows = torch.empty((Cn * N, SURFEL_ROW), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        ws = _bytes(lib.gsb_2dgs_batch_workspace_bytes(Cn, N, H, W, 0), dev)
        _lib.check(lib.gsb_2dgs_batch_backward_geometry(
            Cn, H, W, N, P, _ptr(records), _ptr(contrib), _ptr(final_tau), _ptr(ranges), _ptr(gsid),
            *[_ptr(t) for t in planes[:4]], _ptr(ws), ws.numel(), _ptr(rows), near, far, _ptr(alpha), _ptr(moments),
            _ptr(median_contrib), *[_ptr(t) for t in planes[4:6]], _stream()), lib)
    return rows


# ---------------------------------------------------------------------------------------
# Mesh extraction (gsb_tsdf_*, DESIGN 3.17): projective TSDF fusion of depth maps and marching
# cubes.  The grid: point (i, j, k) at origin + voxel_size (i, j, k); tsdf, weight [nz, ny, nx] and
# color_grid [3, nz, ny, nx] (or None), float32 CUDA tensors, contiguous (updated in place).
def _tsdf_grid(tsdf, weight, color_grid, origin, voxel_size):
    """checks the volume tensors and geometry -> (nx, ny, nz, ox, oy, oz, voxel)"""
    for t, name in ((tsdf, "tsdf"), (weight, "weight")):
        _chk(t, name, ndim=3)
        if not t.is_contiguous():
            raise ValueError("%s must be contiguous (it is updated in place)" % name)
    if weight.shape != tsdf.shape:
        raise ValueError("weight must have the shape of tsdf %s, got %s" % (tuple(tsdf.shape), tuple(weight.shape)))
    _same_device(tsdf, weight)
    nz, ny, nx = tsdf.shape
    if color_grid is not None:
        _chk(color_grid, "color_grid", ndim=4)
        if not color_grid.is_contiguous() or color_grid.shape != (3, nz, ny, nx):
            raise ValueError("color_grid must be a contiguous [3, nz, ny, nx] tensor")
        _same_device(tsdf, color_grid)
    origin = [float(x) for x in origin]
    if len(origin) != 3:
        raise ValueError("origin must have 3 values")
    return (nx, ny, nz, *origin, float(voxel_size))


def tsdf_integrate(tsdf, weight, color_grid, origin, voxel_size, trunc, depth_trunc, cams, depth, color=None):
    """Fuses V depth maps into the volume in place, in view order (gsb_tsdf_integrate): cams is a
    [V, 20] camera table (`camera_table`, pinhole), depth [V, H, W] and color [V, 3, H, W] float32
    CUDA tensors; color with color_grid only.  A depth that is not finite, <= 0 or > depth_trunc
    leaves its points alone.  One call with V views gives bit-identical grids to V calls."""
    grid = _tsdf_grid(tsdf, weight, color_grid, origin, voxel_size)
    cams = _chk(cams, "cams", last=CAMERA_ROW, ndim=2)
    depth = _chk(depth, "depth", ndim=3)
    V, H, W = depth.shape
    if cams.shape[0] != V:
        raise ValueError("cams must have one row per depth map")
    size = cams[:, 16:18].cpu()  # the table's W, H: intrinsics for another resolution would be fused silently
    if not (size == torch.tensor([float(W), float(H)])).all():
        raise ValueError("the camera table's width and height must be the depth map's %dx%d, got %s"
                         % (W, H, size.tolist()))
    if (color is None) != (color_grid is None):
        raise ValueError("color and color_grid go together: pass both or neither")
    if color is not None:
        color = _chk(color, "color", ndim=4)
        if color.shape != (V, 3, H, W):
            raise ValueError("color must be [V, 3, H, W] = %s, got %s" % ((V, 3, H, W), tuple(color.shape)))
    _same_device(tsdf, cams, depth, *([color] if color is not None else []))
    lib = _L()
    with torch.cuda.device(tsdf.device):
        _lib.check(lib.gsb_tsdf_integrate(*grid, float(trunc), float(depth_trunc), V, H, W, _ptr(cams), _ptr(depth),
                                          _ptr(color), _ptr(tsdf), _ptr(weight), _ptr(color_grid), _stream()), lib)


def tsdf_extract(tsdf, weight, color_grid, origin, voxel_size):
    """Marching cubes over the observed part of the volume (gsb_tsdf_extract_*): -> (verts[V, 3]
    float32, faces[F, 3] int32, colors[V, 3] float32 or None), deterministic.  Waits for the
    counts on the host once."""
    grid = _tsdf_grid(tsdf, weight, color_grid, origin, voxel_size)
    nx, ny, nz = grid[:3]
    lib = _L()
    dev = tsdf.device
    ws = _bytes(max(int(lib.gsb_tsdf_extract_workspace_bytes(nx, ny, nz)), 256), dev)
    counts = (C.c_int64 * 2)()
    with torch.cuda.device(dev):
        _lib.check(lib.gsb_tsdf_extract_plan(nx, ny, nz, _ptr(tsdf), _ptr(weight), _ptr(ws), ws.numel(), counts,
                                             _stream()), lib)
        nv, nf = int(counts[0]), int(counts[1])
        verts = torch.empty((nv, 3), dtype=torch.float32, device=dev)
        faces = torch.empty((nf, 3), dtype=torch.int32, device=dev)
        colors = torch.empty((nv, 3), dtype=torch.float32, device=dev) if color_grid is not None else None
        _lib.check(lib.gsb_tsdf_extract_emit(*grid, _ptr(tsdf), _ptr(weight), _ptr(color_grid), _ptr(ws), ws.numel(),
                                             nv, nf, _ptr(verts), _ptr(colors), _ptr(faces), _stream()), lib)
    return verts, faces, colors


# ---------------------------------------------------------------------------------------
# Bilateral-grid colour correction (gsb_bilagrid_*, DESIGN 3.20).  grids[M, 12, L, Y, X] float32,
# channel 4 r + k = A[r][k] of a 3 x 4 affine colour matrix; rgb is one planar image [3, H, W] with
# one grid index, or a batch [B, 3, H, W] with B indices.  Indices are host integers: an int, a
# sequence of ints or a CPU tensor; a CUDA tensor is refused, so no index is ever read back from
# the device and none can reach the kernels unchecked.
BILAGRID_MAX_DIM = 64
BILAGRID_MAX_BATCH = 64


def _bilagrid_dims(shape):
    """checks a grids shape [M, 12, L, Y, X] -> (M, L, Y, X)"""
    if len(shape) != 5 or shape[1] != 12 or shape[0] < 1 or min(shape[2:]) < 1 or max(shape[2:]) > BILAGRID_MAX_DIM:
        raise ValueError("grids must be [M, 12, L, Y, X] with M >= 1 and 1 <= L, Y, X <= %d, got %s"
                         % (BILAGRID_MAX_DIM, tuple(shape)))
    return (int(shape[0]),) + tuple(int(d) for d in shape[2:])


def _bilagrid_shape(grids):
    """checks grids -> (grids contiguous, (M, L, Y, X))"""
    grids = _chk(grids, "grids", ndim=5)
    return grids, _bilagrid_dims(grids.shape)


def _bilagrid_images(rgb, name, image_ids, M):
    """rgb [3,H,W] or [B,3,H,W] and its grid indices -> (rgb contiguous, B, H, W, ids as c_int32[B])"""
    rgb = _chk(rgb, name)
    if rgb.dim() not in (3, 4) or rgb.shape[-3] != 3:
        raise ValueError("%s must be [3, H, W] or [B, 3, H, W], got %s" % (name, tuple(rgb.shape)))
    B = 1 if rgb.dim() == 3 else rgb.shape[0]
    if isinstance(image_ids, torch.Tensor):
        if image_ids.is_cuda:
            raise TypeError("image_ids must be host integers, not a CUDA tensor")
        image_ids = image_ids.reshape(-1).tolist()
    ids = [image_ids] if isinstance(image_ids, numbers.Integral) else list(image_ids)
    if not all(isinstance(i, numbers.Integral) and not isinstance(i, bool) for i in ids):
        raise TypeError("image_ids must be integers")
    if len(ids) != B:
        raise ValueError("%d image ids for a batch of %d images" % (len(ids), B))
    if not 1 <= B <= BILAGRID_MAX_BATCH:
        raise ValueError("the batch must hold 1 to %d images, got %d" % (BILAGRID_MAX_BATCH, B))
    if not all(0 <= i < M for i in ids):
        raise ValueError("image ids must lie in [0, %d), got %s" % (M, ids))
    return rgb, B, rgb.shape[-2], rgb.shape[-1], (C.c_int32 * B)(*[int(i) for i in ids])


def bilagrid_slice(grids, rgb, image_ids):
    """out = A rgb + b per pixel, A read from grids[image_ids[b]] at the pixel's position and
    luminance (gsb_bilagrid_slice) -> a tensor shaped like rgb"""
    grids, shape = _bilagrid_shape(grids)
    rgb, B, H, W, ids = _bilagrid_images(rgb, "rgb", image_ids, shape[0])
    _same_device(grids, rgb)
    out = torch.empty_like(rgb)
    lib = _L()
    with torch.cuda.device(grids.device):
        _lib.check(lib.gsb_bilagrid_slice(*shape, _ptr(grids), B, ids, H, W, _ptr(rgb), _ptr(out), _stream()), lib)
    return out


def bilagrid_sliceB(grids, rgb, image_ids, dloss_dout, dloss_dgrids=None):
    """The slice's backward (gsb_bilagrid_slice_backward) -> (dloss_drgb shaped like rgb,
    dloss_dgrids [M, 12, L, Y, X]).  dloss_dgrids: None (a zeroed tensor is made), or a contiguous
    float32 tensor of grids' shape that the grid gradient is ADDED to."""
    grids, shape = _bilagrid_shape(grids)
    rgb, B, H, W, ids = _bilagrid_images(rgb, "rgb", image_ids, shape[0])
    dout = _chk(dloss_dout, "dloss_dout")
    if dout.shape != rgb.shape:
        raise ValueError("dloss_dout must have rgb's shape %s, got %s" % (tuple(rgb.shape), tuple(dout.shape)))
    if dloss_dgrids is None:
        dloss_dgrids = torch.zeros_like(grids)
    else:
        _chk(dloss_dgrids, "dloss_dgrids")
        if dloss_dgrids.shape != grids.shape or not dloss_dgrids.is_contiguous():
            raise ValueError("dloss_dgrids must be a contiguous tensor of grids' shape (it is added to)")
    _same_device(grids, rgb, dout, dloss_dgrids)
    drgb = torch.empty_like(rgb)
    lib = _L()
    with torch.cuda.device(grids.device):
        _lib.check(lib.gsb_bilagrid_slice_backward(*shape, _ptr(grids), B, ids, H, W, _ptr(rgb), _ptr(dout),
                                                   _ptr(drgb), _ptr(dloss_dgrids), _stream()), lib)
    return drgb, dloss_dgrids


def bilagrid_tv(grids, want_grad=True):
    """Total variation of the grids (gsb_bilagrid_tv): sum over the axes L, Y, X of the mean squared
    difference of neighbours along that axis -> (value [1], dTV/dgrids or None)"""
    grids, shape = _bilagrid_shape(grids)
    lib = _L()
    tv = torch.empty((1,), dtype=torch.float32, device=grids.device)
    grad = torch.empty_like(grids) if want_grad else None
    ws = _bytes(int(lib.gsb_bilagrid_tv_workspace_bytes(*shape)), grids.device)
    with torch.cuda.device(grids.device):
        _lib.check(lib.gsb_bilagrid_tv(*shape, _ptr(grids), _ptr(tv), _ptr(grad), _ptr(ws), ws.numel(), _stream()),
                   lib)
    return tv, grad


# ----------------------------------------------------------------------------- compressed export
KMEANS_MAX_DIM = 64


def _rows(x, name):
    """x: a float32 CUDA [N, D] tensor, 1 <= D <= 64, whose rows may sit any whole number of floats
    apart (a column slice of a wider tensor is read in place) -> (x, row stride in floats)"""
    if not isinstance(x, torch.Tensor):
        raise TypeError("%s must be a torch.Tensor" % name)
    if not x.is_cuda:
        raise ValueError("%s must be a CUDA tensor (there is no CPU path)" % name)
    if x.dtype != torch.float32:
        raise TypeError("%s must be torch.float32, got %s" % (name, x.dtype))
    if x.dim() != 2 or not 1 <= x.shape[1] <= KMEANS_MAX_DIM:
        raise ValueError("%s must be [N, D] with 1 <= D <= %d, got %s" % (name, KMEANS_MAX_DIM, tuple(x.shape)))
    if x.shape[1] > 1 and x.stride(1) != 1 or x.shape[0] > 1 and x.stride(0) < x.shape[1]:
        x = x.contiguous()
    return x, (x.stride(0) if x.shape[0] > 1 else x.shape[1])


def kmeans_assign(x, centroids):
    """The nearest centroid of every row of x[N, D] (gsb_kmeans_assign): a fused distance + argmin
    that never forms the N x K distance matrix; ties go to the lowest index and the result is the
    same bits on every run.  -> (labels int32 [N], squared distances float32 [N])"""
    x, ldx = _rows(x, "x")
    c = _chk(centroids, "centroids", ndim=2)
    _same_device(x, c)
    N, D = x.shape
    K = c.shape[0]
    if c.shape[1] != D or K < 1:
        raise ValueError("centroids must be [K >= 1, %d], got %s" % (D, tuple(c.shape)))
    labels = torch.empty((N,), dtype=torch.int32, device=x.device)
    dist = torch.empty((N,), dtype=torch.float32, device=x.device)
    lib = _L()
    ws = _bytes(int(lib.gsb_kmeans_assign_workspace_bytes(K, D)), x.device)
    with torch.cuda.device(x.device):
        _lib.check(lib.gsb_kmeans_assign(N, K, D, _ptr(x), ldx, _ptr(c), _ptr(labels), _ptr(dist), _ptr(ws),
                                         ws.numel(), _stream()), lib)
    return labels, dist


def kmeans_update(x, labels, centroids):
    """One Lloyd update (gsb_kmeans_update): each centroid becomes the mean of the rows of x[N, D]
    labelled with it, summed in fp64 in ascending row index; an empty cluster keeps its centroid bit
    for bit.  labels: int32 [N] in [0, K).  -> (centroids float32 [K, D], counts int32 [K])"""
    x, ldx = _rows(x, "x")
    c = _chk(centroids, "centroids", ndim=2)
    labels = _chk(labels, "labels", dtype=torch.int32, ndim=1)
    _same_device(x, c, labels)
    N, D = x.shape
    K = c.shape[0]
    if c.shape[1] != D or K < 1:
        raise ValueError("centroids must be [K >= 1, %d], got %s" % (D, tuple(c.shape)))
    if labels.shape[0] != N:
        raise ValueError("labels must have N = %d elements, got %d" % (N, labels.shape[0]))
    perm = torch.sort(labels, stable=True).indices.to(torch.int32)
    out = torch.empty_like(c)
    counts = torch.empty((K,), dtype=torch.int32, device=x.device)
    lib = _L()
    with torch.cuda.device(x.device):
        _lib.check(lib.gsb_kmeans_update(N, K, D, _ptr(x), ldx, _ptr(labels), _ptr(perm), _ptr(c), _ptr(out),
                                         _ptr(counts), _stream()), lib)
    return out, counts


def quantize(x, bits, log_transform=False, value_range=None):
    """Per-column scalar quantisation of x[N, D] (gsb_quantize) to `bits` (8 or 16) bit codes:
    q = clamp(floor((t - lo) (2^bits - 1) / (hi - lo) + 1/2)) of t = x, or sign(x) log1p(|x|) with
    log_transform.  value_range: None (lo, hi = each column's min and max of t, reduced on the device)
    or a float32 [2, D] tensor (lo row, hi row) to use instead.
    -> (codes uint8 / uint16 [N, D], range float32 [2, D])"""
    if bits not in (8, 16):
        raise ValueError("bits must be 8 or 16, got %r" % (bits,))
    x, ldx = _rows(x, "x")
    N, D = x.shape
    if value_range is None:
        rng = torch.empty((2, D), dtype=torch.float32, device=x.device)
    else:
        rng = _chk(value_range, "value_range", ndim=2).clone()
        _same_device(x, rng)
        if tuple(rng.shape) != (2, D):
            raise ValueError("value_range must be [2, %d], got %s" % (D, tuple(rng.shape)))
    codes = torch.empty((N, D), dtype=torch.uint8 if bits == 8 else torch.uint16, device=x.device)
    lib = _L()
    with torch.cuda.device(x.device):
        _lib.check(lib.gsb_quantize(N, D, _ptr(x), ldx, bits, int(bool(log_transform)), int(value_range is None),
                                    _ptr(rng), _ptr(codes), _stream()), lib)
    return codes, rng


def dequantize(codes, value_range, log_transform=False):
    """The inverse of `quantize` (gsb_dequantize): lo + q (hi - lo) / (2^bits - 1), then the inverse
    of the log transform.  codes: uint8 or uint16 [N, D]; value_range: float32 [2, D].
    -> float32 [N, D]"""
    if not isinstance(codes, torch.Tensor) or codes.dtype not in (torch.uint8, torch.uint16):
        raise TypeError("codes must be a uint8 or uint16 tensor")
    if not codes.is_cuda:
        raise ValueError("codes must be a CUDA tensor (there is no CPU path)")
    if codes.dim() != 2 or not 1 <= codes.shape[1] <= KMEANS_MAX_DIM:
        raise ValueError("codes must be [N, D] with 1 <= D <= %d, got %s" % (KMEANS_MAX_DIM, tuple(codes.shape)))
    codes = codes.contiguous()
    N, D = codes.shape
    rng = _chk(value_range, "value_range", ndim=2)
    _same_device(codes, rng)
    if tuple(rng.shape) != (2, D):
        raise ValueError("value_range must be [2, %d], got %s" % (D, tuple(rng.shape)))
    out = torch.empty((N, D), dtype=torch.float32, device=codes.device)
    lib = _L()
    with torch.cuda.device(codes.device):
        _lib.check(lib.gsb_dequantize(N, D, _ptr(codes), 8 if codes.dtype == torch.uint8 else 16, _ptr(rng),
                                      int(bool(log_transform)), _ptr(out), _stream()), lib)
    return out
