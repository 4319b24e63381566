"""ctypes/numpy front-end of the CPU oracle (oracle/gs_oracle.c).  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / `--impl reference` leg
may import this module.  Nothing under easygaussiansplatting_b200/ or gsplatcu/ does.

Every function takes the same float32 arrays the GPU op takes and returns float64 values
(int32 for integer outputs).  Reference citations live next to each C function.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libgs_oracle.so")
_lib = None


def build(force=False):
    """Compile gs_oracle.c with the Makefile next to it (gcc -O2 -fopenmp)."""
    src = os.path.join(_HERE, "gs_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.run(["make", "-C", _HERE, "-s"] + (["-B"] if force else []), check=True)
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_SO)
        _lib.orc_bin.restype = C.c_int64
        _lib.orc_num_threads.restype = C.c_int
    return _lib


def num_threads():
    return int(lib().orc_num_threads())


def set_num_threads(n):
    """OpenMP threads of every later call (bench.py: os.cpu_count(), whatever OMP_NUM_THREADS says)."""
    lib().orc_set_num_threads(int(n))


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f(x):
    return C.c_float(float(x))


# ---------------------------------------------------------------- per-Gaussian stages
def project(pws, Rcw, tcw, fx, fy, cx, cy, calc_J=True):
    """kernel.cu:553-617.  -> us[N,2], pcs[N,3], depths[N] (f64; -1 = culled), du_dpcs[N,2,3]"""
    pws, Rcw, tcw = _f32(pws), _f32(Rcw), _f32(tcw)
    N = pws.shape[0]
    us = np.empty((N, 2)); pcs = np.empty((N, 3)); depths = np.empty(N)
    J = np.empty((N, 2, 3)) if calc_J else None
    lib().orc_project(N, _p(pws), _p(Rcw), _p(tcw), _f(fx), _f(fy), _f(cx), _f(cy),
                      _p(us), _p(pcs), _p(depths), _p(J))
    return (us, pcs, depths, J) if calc_J else (us, pcs, depths)


def compute_cov3d(rots, scales, depths, calc_J=True):
    """kernel.cu:326-423.  -> cov3ds[N,6], dcov3d_drots[N,6,4], dcov3d_dscales[N,6,3]"""
    rots, scales, depths = _f32(rots), _f32(scales), _f32(depths)
    N = rots.shape[0]
    cov = np.empty((N, 6))
    Jr = np.empty((N, 6, 4)) if calc_J else None
    Js = np.empty((N, 6, 3)) if calc_J else None
    lib().orc_cov3d(N, _p(rots), _p(scales), _p(depths), _p(cov), _p(Jr), _p(Js))
    return (cov, Jr, Js) if calc_J else (cov,)


def compute_cov2d(cov3ds, pcs, Rcw, depths, fx, fy, width, height, calc_J=True,
                  return_clamped=False):
    """kernel.cu:425-551.  -> cov2ds[N,3], dcov2d_dcov3ds[N,3,6], dcov2d_dpcs[N,3,3]"""
    cov3ds, pcs, Rcw, depths = _f32(cov3ds), _f32(pcs), _f32(Rcw), _f32(depths)
    N = pcs.shape[0]
    cov = np.empty((N, 3))
    Jc = np.empty((N, 3, 6)) if calc_J else None
    Jp = np.empty((N, 3, 3)) if calc_J else None
    cl = np.zeros(N, dtype=np.uint8)
    lib().orc_cov2d(N, _p(cov3ds), _p(pcs), _p(Rcw), _p(depths), _f(fx), _f(fy), _f(width),
                    _f(height), _p(cov), _p(Jc), _p(Jp), _p(cl))
    out = (cov, Jc, Jp) if calc_J else (cov,)
    return out + (cl.astype(bool),) if return_clamped else out


def sh2color(shs, pws, twc, calc_J=True):
    """kernel.cu:619-807.  -> colors[N,3], dcolor_dshs[N,1,k], dcolor_dpws[N,3,3]"""
    shs, pws, twc = _f32(shs), _f32(pws), _f32(twc)
    N, k = shs.shape[0], shs.shape[1] // 3
    col = np.empty((N, 3))
    Js = np.empty((N, 1, k)) if calc_J else None
    Jp = np.empty((N, 3, 3)) if calc_J else None
    lib().orc_sh2color(N, k, _p(shs), _p(pws), _p(twc), _p(col), _p(Js), _p(Jp))
    return (col, Js, Jp) if calc_J else (col,)


def inverse_cov2d(cov2ds, depths, calc_J=True):
    """kernel.cu:274-324.  depths: float32 array, MODIFIED IN PLACE (NaN det -> -1).
    -> cinv2ds[N,3] f64, areas[N,2] i32, dcinv2d_dcov2ds[N,3,3]"""
    cov2ds = _f32(cov2ds)
    assert depths.dtype == np.float32 and depths.flags.c_contiguous
    N = cov2ds.shape[0]
    cinv = np.empty((N, 3)); areas = np.empty((N, 2), dtype=np.int32)
    J = np.empty((N, 3, 3)) if calc_J else None
    lib().orc_inv_cov2d(N, _p(cov2ds), _p(depths), _p(cinv), _p(areas), _p(J))
    return (cinv, areas, J) if calc_J else (cinv, areas)


# ---------------------------------------------------------------- splat / splatB
def bin(height, width, us, depths, areas):
    """gausplat.cu:50-91 + kernel.cu:46-150: the binning alone (no compositing, so large frames
    stay cheap).  depths (f32) and areas (i32) are MODIFIED IN PLACE like the device op.
    -> (P, ranges[T,2] i32, gsid[P] i32, keys[P] u64 as (tile << 32 | depth key))"""
    us = _f32(us)
    assert depths.dtype == np.float32 and depths.flags.c_contiguous
    assert areas.dtype == np.int32 and areas.flags.c_contiguous
    N = us.shape[0]
    H, W = int(height), int(width)
    T = ((W + 15) // 16) * ((H + 15) // 16)
    L = lib()
    P = int(L.orc_bin(H, W, N, _p(us), _p(depths), _p(areas), None, None, None))
    ranges = np.zeros((T, 2), dtype=np.int32)
    gsid = np.empty(max(P, 1), dtype=np.int32)
    keys = np.empty(max(P, 1), dtype=np.uint64)
    L.orc_bin(H, W, N, _p(us), _p(depths), _p(areas), _p(ranges), _p(gsid), _p(keys))
    return P, ranges, gsid[:P], keys[:P]


def splat(height, width, us, cinv2ds, alphas, depths, colors, areas, margin=2e-5):
    """gausplat.cu:24-112 + kernel.cu:46-271.  depths (f32) and areas (i32) are MODIFIED IN
    PLACE like the device op.  Returns dict(image[3,H,W] f64, contrib[H,W] i32,
    final_tau[H,W] f64, ranges[T,2] i32, gsid[P] i32, keys[P] u64, ambiguous[H,W] bool)."""
    us, cinv2ds, colors = _f32(us), _f32(cinv2ds), _f32(colors)
    alphas = _f32(alphas).reshape(-1)
    H, W = int(height), int(width)
    P, ranges, gsid, keys = bin(H, W, us, depths, areas)
    L = lib()
    image = np.empty((3, H, W)); contrib = np.empty((H, W), dtype=np.int32)
    ftau = np.empty((H, W)); amb = np.empty((H, W), dtype=np.uint8)
    L.orc_draw(H, W, _p(ranges), _p(gsid), _p(us), _p(cinv2ds), _p(alphas), _p(colors),
               _p(image), _p(contrib), _p(ftau), _p(amb), C.c_double(margin))
    return dict(image=image, contrib=contrib, final_tau=ftau, ranges=ranges, gsid=gsid,
                keys=keys, ambiguous=amb.astype(bool), P=int(P))


def splat_backward(height, width, us, cinv2ds, alphas, colors, fwd, dloss_dgammas,
                   return_ambiguous=False, margin=2e-5):
    """kernel.cu:809-950 on the oracle's own forward state `fwd` (dict from splat()).
    -> dloss_dus[N,1,2], dloss_dcinv2ds[N,1,3], dloss_dalphas[N,1,1], dloss_dcolors[N,1,3]
    (+ bool[N]: Gaussians with a replayed alpha' within `margin` of the 0.002 threshold)"""
    us, cinv2ds, colors = _f32(us), _f32(cinv2ds), _f32(colors)
    alphas = _f32(alphas).reshape(-1)
    dl = _f32(dloss_dgammas)
    N = us.shape[0]
    du = np.empty((N, 1, 2)); dc = np.empty((N, 1, 3)); da = np.empty((N, 1, 1))
    dcol = np.empty((N, 1, 3))
    amb = np.zeros(max(N, 1), dtype=np.uint8)[:N]
    lib().orc_drawB(int(height), int(width), N, _p(fwd["ranges"]), _p(fwd["gsid"]), _p(us),
                    _p(cinv2ds), _p(alphas), _p(colors), _p(fwd["final_tau"]),
                    _p(fwd["contrib"]), _p(dl), _p(du), _p(dc), _p(da), _p(dcol), _p(amb),
                    C.c_double(margin))
    return (du, dc, da, dcol, amb.astype(bool)) if return_ambiguous else (du, dc, da, dcol)


MOMENT_COLS = [0, 1, 2, 3, 4, 5, 8, 9, 10]  # the nine moment rows of the colour frame in drawB_rows' columns


def drawB_rows(height, width, us, cinv2ds, alphas, values, fwd, dl_planes, margin=2e-5):
    """orc_drawB_rows: orc_drawB's replay with nch channels (values[N,nch], dl_planes[nch,H,W]) on the
    forward state `fwd`.  -> (rows, abs_rows, maha_rows, amb_rows) [N, 8 + nch] f64 and the bool[N] flags
    of splat_backward; columns: w dx, w dy, w dx^2, w dx dy, w dy^2, dL/dalpha' g, the AbsGS terms
    |w (A dx + B dy)|, |w (B dx + C dy)|, then wc dl_c per channel (gs_oracle.c)"""
    us, cinv2ds = _f32(us), _f32(cinv2ds)
    alphas, vals, dl = _f32(alphas).reshape(-1), _f32(values), _f32(dl_planes)
    N, nch = vals.shape
    H, W = int(height), int(width)
    assert dl.shape == (nch, H, W)
    out = [np.empty((N, 8 + nch)) for _ in range(4)]
    amb = np.zeros(max(N, 1), dtype=np.uint8)[:N]
    lib().orc_drawB_rows(H, W, N, nch, _p(fwd["ranges"]), _p(fwd["gsid"]), _p(us), _p(cinv2ds), _p(alphas),
                         _p(vals), _p(np.ascontiguousarray(fwd["final_tau"], np.float64)),
                         _p(np.ascontiguousarray(fwd["contrib"], np.int32)), _p(dl), *[_p(a) for a in out], _p(amb),
                         C.c_double(margin))
    return tuple(out) + (amb.astype(bool),)


def rows_dict(raw):
    """drawB_rows' output -> dict(rows[N,9], abs_rows, maha_rows, amb_rows, ambiguous bool[N]) in the moment-row
    layout k_draw_bwd writes, plus raw: the [N, 8 + nch] arrays"""
    c = MOMENT_COLS
    R, Ab, Mh, Am, amb = raw
    return dict(rows=R[:, c], abs_rows=Ab[:, c], maha_rows=Mh[:, c], amb_rows=Am[:, c], ambiguous=amb, raw=raw)


def splat_backward_rows(height, width, us, cinv2ds, alphas, colors, fwd, dloss_dgammas, margin=2e-5):
    """The moment rows k_draw_bwd writes (`splatB(..., moments_only=True)`), in fp64, with their conditioning.
    -> rows_dict: rows[N,9] are w dx, w dy, w dx^2, w dx dy, w dy^2, dL/dalpha' g, wc dL/dgamma_rgb
    (DESIGN 3.2); abs_rows the same sums over the magnitudes of every product in a term, maha_rows the
    effect of the exponents' rounding, amb_rows the most a threshold decision within `margin` can move
    an entry (gs_oracle.c)"""
    return rows_dict(drawB_rows(height, width, us, cinv2ds, alphas, colors, fwd, dloss_dgammas, margin))


def moments_to_grads(rows, cinv2ds):
    """k_finalize_grads' conversion in fp64: rows[N,9] -> du[N,2], dconic[N,3], dalpha[N], dcolour[N,3]"""
    m = np.asarray(rows, np.float64)
    c = np.asarray(cinv2ds, np.float64)
    A, B, Cc = c[:, 0], c[:, 1], c[:, 2]
    du = -np.stack([A * m[:, 0] + B * m[:, 1], B * m[:, 0] + Cc * m[:, 1]], 1)
    dc = np.stack([-0.5 * m[:, 2], -m[:, 3], -0.5 * m[:, 4]], 1)
    return du, dc, m[:, 5].copy(), m[:, 6:9].copy()


def moments_to_grads_bound(bound_rows, cinv2ds):
    """the same conversion applied to a conditioning row (abs / maha / amb, >= 0): |A| b0 + |B| b1 for du.x
    and so on -> du[N,2], dconic[N,3], dalpha[N], dcolour[N,3]"""
    b = np.asarray(bound_rows, np.float64)
    c = np.abs(np.asarray(cinv2ds, np.float64))
    du = np.stack([c[:, 0] * b[:, 0] + c[:, 1] * b[:, 1], c[:, 1] * b[:, 0] + c[:, 2] * b[:, 1]], 1)
    return du, np.stack([0.5 * b[:, 2], b[:, 3], 0.5 * b[:, 4]], 1), b[:, 5].copy(), b[:, 6:9].copy()


def forward_cpu_splat(height, width, us, cinv2d, alpha, depth, color, areas):
    """gsplat/gausplat.py:185-245 (the forward_cpu.py renderer).  -> image[H,W,3] f64"""
    f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    us, cinv2d, alpha, depth, color = map(f64, (us, cinv2d, alpha, depth, color))
    areas = np.ascontiguousarray(areas, dtype=np.int32)
    img = np.empty((int(height), int(width), 3))
    lib().orc_forward_cpu_splat(int(height), int(width), us.shape[0], _p(us), _p(cinv2d),
                                _p(alpha), _p(depth), _p(color), _p(areas), _p(img))
    return img


# ---------------------------------------------------------------- full chain (fp64)
def chain_backward(Rcw, dloss_dus, dloss_dcinv2ds, dloss_dalphas, dloss_dcolors,
                   du_dpcs, dcov3d_drots, dcov3d_dscales, dcov2d_dcov3ds, dcov2d_dpcs,
                   dcolor_dshs, dcolor_dpws, dcinv2d_dcov2ds, use_numpy=False):
    """gsmodel.py:72-85 == backward_cpu.py:476-484: the Jacobian chain from the four splatB
    grads to parameter grads, in fp64.  Returns dict(pws, shs, alphas, scales, rots, us)."""
    R = np.ascontiguousarray(Rcw, dtype=np.float64)
    f = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    dus, dci, dal, dco = f(dloss_dus), f(dloss_dcinv2ds), f(dloss_dalphas), f(dloss_dcolors)
    if not use_numpy:  # one C pass (orc_chain); the numpy form below is its cross-check
        N, k = dus.shape[0], np.asarray(dcolor_dshs).shape[-1]
        Js = [f(a) for a in (du_dpcs, dcov3d_drots, dcov3d_dscales, dcov2d_dcov3ds, dcov2d_dpcs,
                             dcolor_dshs, dcolor_dpws, dcinv2d_dcov2ds)]
        dpws = np.empty((N, 3)); dshs = np.empty((N, 3 * k)); dsc = np.empty((N, 3)); dro = np.empty((N, 4))
        lib().orc_chain(N, k, _p(R), _p(dus), _p(dci), _p(dal), _p(dco), *[_p(a) for a in Js],
                        _p(dpws), _p(dshs), _p(dsc), _p(dro))
        return dict(pws=dpws, shs=dshs, alphas=dal.reshape(N, 1), scales=dsc, rots=dro,
                    us=dus.reshape(N, 2))
    dcov2d = dci @ f(dcinv2d_dcov2ds)
    dcov3d = dcov2d @ f(dcov2d_dcov3ds)
    drots = dcov3d @ f(dcov3d_drots)
    dscales = dcov3d @ f(dcov3d_dscales)
    dshs = (dco.transpose(0, 2, 1) @ f(dcolor_dshs)).transpose(0, 2, 1)
    dshs = dshs.reshape(dshs.shape[0], -1)
    dpws = dus @ f(du_dpcs) @ R + dco @ f(dcolor_dpws) + dcov2d @ f(dcov2d_dpcs) @ R
    return dict(pws=dpws[:, 0], shs=dshs, alphas=dal[:, 0], scales=dscales[:, 0],
                rots=drots[:, 0], us=dus[:, 0])


# ---------------------------------------------------------------- training loss (row N2)
def ssim_window():
    """gsplat/pytorch_ssim.py:12-15: 11 taps, sigma 1.5, built and normalised in float32"""
    g = np.array([np.exp(-(x - 5) ** 2 / float(2 * 1.5 ** 2)) for x in range(11)], dtype=np.float32)
    return (g / g.sum(dtype=np.float32)).astype(np.float64)


def gau_loss(image, gt, loss_lambda=0.2, want_grad=True):
    """gsplat/pytorch_ssim.py:64-67 (+ its autograd gradient).  image, gt: [3,H,W] float32.
    -> dict(loss, l1, ssim, dloss_dimage[3,H,W] f64)"""
    image, gt = _f32(image), _f32(gt)
    assert image.shape == gt.shape and image.ndim == 3
    Cn, H, W = image.shape
    assert Cn == 3
    win = ssim_window()
    loss, l1, ss = C.c_double(0), C.c_double(0), C.c_double(0)
    grad = np.empty((3, H, W)) if want_grad else None
    lib().orc_gau_loss(H, W, _p(image), _p(gt), C.c_double(loss_lambda), _p(win), C.byref(loss), C.byref(l1),
                       C.byref(ss), _p(grad))
    return dict(loss=loss.value, l1=l1.value, ssim=ss.value, dloss_dimage=grad)
