"""fp64 Mip-Splatting 3D smoothing filter (gsb_filter3d, gsb_filter3d_apply, gsb_filter3d_backward).
TEST INFRASTRUCTURE ONLY.

Filter, for Gaussian i and the training cameras k (rows of the [C, 20] table: Rcw 9, tcw 3, fx, fy,
cx, cy, W, H, 2 unused):
    pc = Rcw pw + tcw,  u = (fx x / z + cx, fy y / z + cy)
    k sees i  iff  z >= 0.2f  and  -0.15 W <= u_x <= 1.15 W  and  -0.15 H <= u_y <= 1.15 H
    d_i = min z over the cameras that see i (the largest d of the seen Gaussians if none does)
    filter3d_i = sqrt(variance) d_i / max_k fx_k      (all 0 when nothing is seen or no fx > 0)
The camera-frame depth z is evaluated as the kernels do (three fp32 fused multiply-adds, emulated
through fp64), so the chosen d_i is an fp32 value the device can reproduce bit for bit; the
visibility decisions are taken on that z and on an fp64 u, and a row whose decision for some camera
lies within a relative 1e-6 of the z or a screen bound is flagged (fp32 may decide it either way).
Apply (f = filter3d_i):  s'_j = sqrt(s_j^2 + f^2),  t_j = s_j / s'_j,  alpha' = t_0 t_1 t_2 alpha
(f == 0: s' = s, alpha' = alpha).  Backward:
    dL/ds_j = dL/ds'_j t_j + alpha dL/dalpha' prod_{k != j} t_k f^2 / s'_j^3,   dL/dalpha = c dL/dalpha'
"""
import numpy as np

MIN_DEPTH = np.float32(0.2)
MARGIN = np.float32(0.15)
HI = np.float32(np.float32(1.0) + MARGIN)  # the fp32 constant 1.15f the kernels compare against


def _fma32(a, b, c):
    """fp32 fmaf(a, b, c) through fp64: the product of two fp32 values is exact there"""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def camera_z(pws, cam):
    """the kernels' fp32 camera-frame depth of every row of pws[N,3] (f32) in camera row `cam`"""
    R, t = cam[:9], cam[9:12]
    return _fma32(R[6], pws[:, 0], _fma32(R[7], pws[:, 1], _fma32(R[8], pws[:, 2], t[2])))


def visibility(pws, cam, rel=1e-6):
    """-> (seen[N], z32[N], flagged[N]) for one camera row"""
    pws = np.asarray(pws, np.float32)
    cam = np.asarray(cam, np.float32)
    z32 = camera_z(pws, cam)
    p64 = pws.astype(np.float64)
    R = cam[:9].astype(np.float64).reshape(3, 3)
    pc = p64 @ R.T + cam[9:12].astype(np.float64)
    fx, fy, cx, cy = (float(v) for v in cam[12:16])
    W, H = cam[16], cam[17]
    kept = z32 >= MIN_DEPTH
    flag = np.abs(pc[:, 2] - 0.2) <= rel * 0.2
    with np.errstate(divide="ignore", invalid="ignore"):
        zs = np.where(kept, pc[:, 2], 1.0)
        px, py = fx * pc[:, 0] / zs, fy * pc[:, 1] / zs
    ux, uy = px + cx, py + cy
    seen = kept.copy()
    for u, mag, lo, hi in ((ux, np.abs(px) + abs(cx), -MARGIN * W, HI * W), (uy, np.abs(py) + abs(cy), -MARGIN * H,
                                                                             HI * H)):
        lo, hi = float(lo), float(hi)  # the fp32 bounds
        seen &= (u >= lo) & (u <= hi)
        tol = rel * (mag + max(abs(lo), abs(hi)))
        flag |= kept & ((np.abs(u - lo) <= tol) | (np.abs(u - hi) <= tol))
    return seen, z32, flag


def filter3d(pws, table, variance=0.2):
    """-> dict(filter[N] f64, d[N] (the fp32 d_i as f64; the fallback for unseen rows), seen[N] (by
    some camera), flagged[N], fmax, dmax)"""
    pws = np.asarray(pws, np.float32)
    table = np.asarray(table, np.float32).reshape(-1, 20)
    N = pws.shape[0]
    best = np.full(N, np.inf, np.float32)
    flagged = np.zeros(N, bool)
    for cam in table:
        seen, z32, flag = visibility(pws, cam)
        best = np.where(seen, np.minimum(best, z32), best)
        flagged |= flag
    seen = np.isfinite(best)
    fmax = max(float(np.nanmax(table[:, 12])), 0.0) if len(table) else 0.0  # the largest positive fx
    dmax = float(best[seen].max()) if seen.any() else 0.0
    d = np.where(seen, best.astype(np.float64), dmax)
    f = np.sqrt(float(np.float32(variance))) * d / fmax if dmax > 0 and fmax > 0 else np.zeros(N)
    return dict(filter=f, d=d, seen=seen, flagged=flagged, fmax=fmax, dmax=dmax)


def apply(scales, alphas, f):
    """-> (scales_f[N,3], alphas_f[N], t[N,3]) in fp64"""
    s = np.asarray(scales, np.float64).reshape(-1, 3)
    a = np.asarray(alphas, np.float64).reshape(-1)
    f = np.asarray(f, np.float64).reshape(-1, 1)
    sf = np.sqrt(s * s + f * f)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.where(f == 0, 1.0, s / sf)
    sf = np.where(f == 0, s, sf)
    return sf, t.prod(1) * a, t


def backward(scales, alphas, f, dloss_dscales_f, dloss_dalphas_f):
    """-> (dL/ds[N,3], dL/dalpha[N]) in fp64"""
    s = np.asarray(scales, np.float64).reshape(-1, 3)
    a = np.asarray(alphas, np.float64).reshape(-1)
    fr = np.asarray(f, np.float64).reshape(-1, 1)
    gsf = np.asarray(dloss_dscales_f, np.float64).reshape(-1, 3)
    gaf = np.asarray(dloss_dalphas_f, np.float64).reshape(-1)
    sf, _, t = apply(s, a, fr)
    other = np.stack([t[:, 1] * t[:, 2], t[:, 0] * t[:, 2], t[:, 0] * t[:, 1]], axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        k = np.where(fr == 0, 0.0, fr * fr / sf ** 3)
    gs = gsf * t + (a * gaf)[:, None] * other * k
    return gs, t.prod(1) * gaf
