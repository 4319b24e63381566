"""fp64 OpenCV radial-tangential camera model (COLMAP's OPENCV, RADIAL, SIMPLE_RADIAL) of the per-Gaussian
stages.  TEST INFRASTRUCTURE ONLY.  DESIGN 3.19 states the model; camera_model_oracle holds the others, and
every function here takes the same arguments and passes any other model through to it.

With (a, b) = (x/z, y/z), rho = a^2 + b^2, R = 1 + k1 rho + k2 rho^2 and k = (k1, k2, p1, p2):
    delta(a, b) = (a R + 2 p1 a b + p2 (rho + 2 a^2),  b R + p1 (rho + 2 b^2) + 2 p2 a b)
    u  = (fx delta_x(a, b) + cx, fy delta_y(a, b) + cy)                            (never clamped)
    J  = diag(f) Ddelta(ah, bh) (1/z) [[1, 0, -ah], [0, 1, -bh]],  (ah, bh) = clamp((a, b), +-lim)
    Ju = the same at the unclamped (a, b): du/dpc, which the chain's dL/du goes through
`opencv_limits` gives lim, `opencv_valid` the cull (rho < rho_valid and det Ddelta(a, b) > 0).  `stages`,
`camera_grad` and `step` compose with oracle.chain_backward, aa_oracle, rgbd_oracle and the rasterizer
oracles as camera_model_oracle's do.
"""
import numpy as np

from . import camera_model_oracle as ocm
from . import filter3d_oracle as of3
from . import oracle as orc
from . import rgbd_oracle as ordb
from . import step_oracle as ostep

oaa = ocm.oaa
MODELS = ocm.MODELS + ("opencv",)


def _k(k):
    return np.zeros(4) if k is None else np.asarray(k, np.float64).reshape(4)


def opencv_rho_valid(k1, k2):
    """the smallest positive root of d(r R)/dr = 1 + 3 k1 rho + 5 k2 rho^2 (inf if none)"""
    if k1 == 0 and k2 == 0:
        return np.inf
    roots = np.roots([5.0 * k2, 3.0 * k1, 1.0] if k2 != 0 else [3.0 * k1, 1.0])
    pos = [r.real for r in np.atleast_1d(roots) if abs(r.imag) <= 1e-12 * max(1.0, abs(r.real)) and r.real > 0]
    return min(pos) if pos else np.inf


def _solve_radial(rd, k1, k2):
    """r_u with r_u (1 + k1 r_u^2 + k2 r_u^4) = rd below sqrt(rho_valid) (sqrt(rho_valid) beyond the maximum)"""
    from scipy.optimize import brentq
    dist = lambda r: r * (1 + r * r * (k1 + r * r * k2))
    rv = opencv_rho_valid(k1, k2)
    if np.isfinite(rv) and dist(np.sqrt(rv)) <= rd:
        return np.sqrt(rv)
    hi = np.sqrt(rv) if np.isfinite(rv) else max(rd, 1e-300)
    while dist(hi) < rd:
        hi *= 2
    return brentq(lambda r: dist(r) - rd, 0.0, hi, xtol=1e-15, rtol=1e-15, maxiter=500)


def opencv_limits(k, fx, fy, cx, cy, width, height):
    """(Lx, Ly) = 1.3 (W / (2 fx), H / (2 fy)) c with c = r_u / r_d: r_d the largest |((u - cx) / fx, (v - cy) / fy)|
    over the four image corners, r_u its undistorted radius (`_solve_radial`).  c = 1 when k1 = k2 = 0; the
    tangential terms are left to the 1.3 margin."""
    k1, k2 = _k(k)[:2]
    c = 1.0
    if k1 != 0 or k2 != 0:
        rd = max(np.hypot((u - cx) / fx, (v - cy) / fy) for u in (0.0, width) for v in (0.0, height))
        c = _solve_radial(rd, k1, k2) / rd
    return 1.3 * width / (2 * fx) * c, 1.3 * height / (2 * fy) * c


def opencv_terms(a, b, k):
    """delta (dx, dy), Ddelta (D00, D01, D11) and its derivatives dD/da, dD/db (each (00, 01, 11)) at (a, b)"""
    k1, k2, p1, p2 = _k(k)
    rho = a * a + b * b
    R, R1, R2 = 1 + rho * (k1 + rho * k2), k1 + 2 * k2 * rho, 2 * k2
    dlt = (a * R + 2 * p1 * a * b + p2 * (rho + 2 * a * a), b * R + p1 * (rho + 2 * b * b) + 2 * p2 * a * b)
    D = (R + 2 * a * a * R1 + 2 * p1 * b + 6 * p2 * a, 2 * a * b * R1 + 2 * p1 * a + 2 * p2 * b,
         R + 2 * b * b * R1 + 6 * p1 * b + 2 * p2 * a)
    Da = (6 * a * R1 + 4 * a ** 3 * R2 + 6 * p2, 2 * b * R1 + 4 * a * a * b * R2 + 2 * p1,
          2 * a * R1 + 4 * a * b * b * R2 + 2 * p2)
    Db = (Da[1], Da[2], 6 * b * R1 + 4 * b ** 3 * R2 + 6 * p1)
    return dlt, D, Da, Db


def _J(a, b, z, fx, fy, D):
    J = np.zeros((len(z), 2, 3))
    for r, f, (d0, d1) in ((0, fx, (D[0], D[1])), (1, fy, (D[1], D[2]))):
        J[:, r, 0], J[:, r, 1], J[:, r, 2] = f * d0 / z, f * d1 / z, -f * (d0 * a + d1 * b) / z
    return J


def opencv_valid(pc, k):
    """-> (valid, (rho_valid - rho) / rho_valid, det Ddelta) at pc[N,3]: valid = rho < rho_valid and det > 0"""
    pc = np.asarray(pc, np.float64).reshape(-1, 3)
    a, b = pc[:, 0] / pc[:, 2], pc[:, 1] / pc[:, 2]
    k4 = _k(k)
    rv = opencv_rho_valid(k4[0], k4[1])
    D = opencv_terms(a, b, k4)[1]
    det = D[0] * D[2] - D[1] * D[1]
    rho = a * a + b * b
    drho = (rv - rho) / rv if np.isfinite(rv) else np.full(len(a), np.inf)
    return (rho < rv) & (det > 0), drho, det


def project(pc, model, fx, fy, cx, cy, k=None, lim=None):
    """camera_model_oracle.project; for "opencv" (k = (k1, k2, p1, p2), lim = (Lx, Ly)) -> u[N,2], the clamped
    J[N,2,3], dJ[N,2,3,3] = dJ[a,b]/dpc[c] (a clamped coordinate has no derivative), valid[N] and
    Ju[N,2,3] = du/dpc (unclamped)"""
    if model != "opencv":
        return ocm.project(pc, model, fx, fy, cx, cy, k)
    pc = np.asarray(pc, np.float64).reshape(-1, 3)
    N = pc.shape[0]
    x, y, z = pc[:, 0], pc[:, 1], pc[:, 2]
    fx, fy, cx, cy = (float(v) for v in (fx, fy, cx, cy))
    a, b = x / z, y / z
    Lx, Ly = lim
    ah, bh = np.clip(a, -Lx, Lx), np.clip(b, -Ly, Ly)
    mx, my = (np.abs(a) <= Lx).astype(np.float64), (np.abs(b) <= Ly).astype(np.float64)
    dlt, Du, _, _ = opencv_terms(a, b, k)
    u = np.stack([fx * dlt[0] + cx, fy * dlt[1] + cy], axis=1)
    Ju = _J(a, b, z, fx, fy, Du)
    _, D, Da, Db = opencv_terms(ah, bh, k)
    J = _J(ah, bh, z, fx, fy, D)
    # J = K(ah, bh) / z;  dah/dx = mx / z, dah/dz = -mx ah / z (the same for bh)
    f = (fx, fy)
    dKa, dKb = np.zeros((N, 2, 3)), np.zeros((N, 2, 3))
    for r, (i0, i1) in ((0, (0, 1)), (1, (1, 2))):
        dKa[:, r, 0], dKa[:, r, 1] = f[r] * Da[i0], f[r] * Da[i1]
        dKa[:, r, 2] = -f[r] * (Da[i0] * ah + D[i0] + Da[i1] * bh)
        dKb[:, r, 0], dKb[:, r, 1] = f[r] * Db[i0], f[r] * Db[i1]
        dKb[:, r, 2] = -f[r] * (Db[i0] * ah + Db[i1] * bh + D[i1])
    dJ = np.zeros((N, 2, 3, 3))
    z2 = (z * z)[:, None, None]
    dJ[..., 0] = dKa * mx[:, None, None] / z2
    dJ[..., 1] = dKb * my[:, None, None] / z2
    dJ[..., 2] = -J / z[:, None, None] - (dKa * (mx * ah)[:, None, None] + dKb * (my * bh)[:, None, None]) / z2
    return u, J, dJ, opencv_valid(pc, k)[0], Ju


def unproject_opencv(u, fx, fy, cx, cy, k=None, iters=60):
    """(a, b)[N,2] with delta(a, b) = ((u - cx) / fx, (v - cy) / fy): Newton on delta from the distorted
    point, each step halved until the residual falls"""
    u = np.asarray(u, np.float64).reshape(-1, 2)
    mx, my = (u[:, 0] - cx) / fx, (u[:, 1] - cy) / fy
    x, y = mx.copy(), my.copy()

    def res(x, y):
        d = opencv_terms(x, y, k)[0]
        return d[0] - mx, d[1] - my

    for _ in range(iters):
        ex, ey = res(x, y)
        D = opencv_terms(x, y, k)[1]
        det = D[0] * D[2] - D[1] * D[1]
        sx, sy = (D[2] * ex - D[1] * ey) / det, (D[0] * ey - D[1] * ex) / det
        t = np.ones_like(x)
        for _ in range(40):
            rx, ry = res(x - t * sx, y - t * sy)
            worse = np.hypot(rx, ry) > np.hypot(ex, ey)
            if not worse.any():
                break
            t = np.where(worse, 0.5 * t, t)
        x, y = x - t * sx, y - t * sy
    return np.stack([x, y], axis=1)


def opencv_band(pc, k, fx, fy, cx, cy, width, height, tol=1e-4):
    """rows of pc[N,3] within tol (relative) of the opencv cull (rho_valid, det Ddelta = 0) or clamp: fp32
    rounding may put them on either side"""
    pc = np.asarray(pc, np.float64).reshape(-1, 3)
    Lx, Ly = opencv_limits(k, *(float(np.float32(v)) for v in (fx, fy, cx, cy)), float(width), float(height))
    _, drho, det = opencv_valid(pc, k)
    a, b = pc[:, 0] / pc[:, 2], pc[:, 1] / pc[:, 2]
    return ((np.abs(drho) < tol) | (np.abs(det) < tol) | (np.abs(np.abs(a) - Lx) < tol * Lx) |
            (np.abs(np.abs(b) - Ly) < tol * Ly))


def stages(pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy, width, height, model="pinhole", k=None):
    """camera_model_oracle.stages; for "opencv" J[0] (the chain's du/dpc) is the unclamped Ju and Jm the
    clamped J of cov2d within `opencv_limits` of the frame.  A Gaussian past the fold is culled like
    z < 0.2 (depth -1)."""
    if model != "opencv":
        return ocm.stages(pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy, width, height, model=model, k=k)
    _, pcs, depths, _ = orc.project(pws, Rcw, tcw, fx, fy, cx, cy)
    pcs = ocm._f32(pcs).astype(np.float64)
    N = pcs.shape[0]
    keep = depths >= 0.2
    pe = np.where(keep[:, None], pcs, np.array([0.0, 0.0, 1.0]))
    f32 = [float(np.float32(v)) for v in (fx, fy, cx, cy)]
    lim = opencv_limits(k, *f32, float(width), float(height))
    u, J, dJ, valid, Jmean = project(pe, "opencv", *f32, k, lim=lim)
    depths = np.where(keep & valid, depths, -1.0)
    d32 = ocm._f32(depths)
    c3, J3r, J3s = orc.compute_cov3d(rots, scales, d32)
    c3 = ocm._f32(c3).astype(np.float64)
    R = ocm._f32(Rcw).astype(np.float64).reshape(3, 3)
    c2, J2c, S = ocm._cov2d(J, R, c3)
    Sp = R[None] @ S @ R.T[None]
    J2p = np.zeros((N, 3, 3))
    for c in range(3):
        X = dJ[:, :, :, c] @ Sp @ J.transpose(0, 2, 1)
        X = X + X.transpose(0, 2, 1)
        J2p[:, 0, c], J2p[:, 1, c], J2p[:, 2, c] = X[:, 0, 0], X[:, 0, 1], X[:, 1, 1]
    col, Jcs, Jcp = orc.sh2color(shs, pws, twc)
    cull = d32 < 0.2
    c2[cull] = 0.0
    ci, areas, Jci = orc.inverse_cov2d(ocm._f32(np.where(cull[:, None], 0.0, c2)), d32)
    kept = d32 >= 0.2  # after the NaN-determinant cull
    Ju = np.where(kept[:, None, None], Jmean, 0.0)
    Jm = np.where(kept[:, None, None], J, 0.0)
    J2c[~kept] = 0.0
    J2p[~kept] = 0.0
    c2[~kept] = 0.0
    us = np.where(kept[:, None], u, 0.0)
    return dict(us=us, ci=ci, col=col, depths=d32, areas=areas, keep=kept, pcs=ocm._f32(pcs), cov3ds=ocm._f32(c3),
                J=(Ju, J3r, J3s, J2c, J2p, Jcs, Jcp, Jci), c2=c2, Jm=Jm, lim=lim)


def camera_grad(st, pws, Rcw, fx, fy, width, height, dloss_dus, dloss_dcinv2ds, dloss_dcolors, dloss_ddepths=None,
                model="pinhole"):
    """camera_model_oracle.camera_grad: dL/du through st["J"][0] (opencv: the unclamped Ju), the direct term
    J^T dL/dM through st["Jm"] (the clamped J)"""
    return ocm.camera_grad(st, pws, Rcw, fx, fy, width, height, dloss_dus, dloss_dcinv2ds, dloss_dcolors,
                           dloss_ddepths, model=model)


def step(scene, cam, *, rgbd, pose, aa, filt, dl, dld=None, dla=None, drawn_inputs=None, model="pinhole", k=None):
    """camera_model_oracle.step; for "opencv" the same composition over this module's `stages`, with the rows
    of `opencv_band` flagged besides step_oracle's"""
    if model != "opencv":
        return ocm.step(scene, cam, rgbd=rgbd, pose=pose, aa=aa, filt=filt, dl=dl, dld=dld, dla=dla,
                        drawn_inputs=drawn_inputs, model=model, k=k)
    H, W = cam["height"], cam["width"]
    if filt is None:
        sf = np.asarray(scene["scales"], np.float64).reshape(-1, 3)
        af = np.asarray(scene["alphas"], np.float64).reshape(-1)
    else:
        sf, af, _ = of3.apply(scene["scales"], scene["alphas"], filt)
    st = stages(scene["pws"], scene["rots"], sf, scene["shs"], cam["Rcw"], cam["tcw"], cam["twc"], cam["fx"],
                cam["fy"], cam["cx"], cam["cy"], W, H, model=model, k=k)
    s = oaa.scale(st["c2"], st["keep"])
    rho = s["rho"] if aa else np.ones(len(af))
    N = len(af)
    inp = drawn_inputs if drawn_inputs is not None else dict(
        us=st["us"], ci=st["ci"], col=st["col"], depths=st["depths"], areas=st["areas"], alphas=rho * af)
    out = ostep.render(cam, rgbd, inp)
    dl = np.asarray(dl, np.float32)
    if rgbd:
        dld = np.zeros((H, W), np.float32) if dld is None else dld
        dla = np.zeros((H, W), np.float32) if dla is None else dla
        du, dc, da, dcol, dz, amb = ordb.splat_backward_rgbd(H, W, inp["us"], inp["ci"], inp["alphas"], inp["col"],
                                                             out["z"], out, dl, dld, dla, return_ambiguous=True)
    else:
        du, dc, da, dcol, amb = orc.splat_backward(H, W, inp["us"], inp["ci"], inp["alphas"], inp["col"], out, dl,
                                                   return_ambiguous=True)
        dz = None
    Rcw = cam["Rcw"]
    ch = orc.chain_backward(Rcw, du, dc, da, dcol, *st["J"])
    da_eff = da.reshape(N)
    gc2 = oaa.dcov2d_addend(st["c2"], st["keep"], af, da_eff) if aa else np.zeros((N, 3))
    g = dict(shs=ch["shs"], us=ch["us"].reshape(N, 2))
    if aa:
        add = oaa.chain(st, Rcw, gc2)
        for key in ("pws", "scales", "rots"):
            g[key] = ch[key] + add[key]
    else:
        g.update(pws=ch["pws"], scales=ch["scales"], rots=ch["rots"])
    if rgbd:
        g["pws"] = g["pws"] + ordb.chain_depth(Rcw, dz, st["depths"])
    dalpha_f = rho * da_eff if aa else da_eff
    if filt is None:
        g["alphas"] = dalpha_f
    else:
        g["scales"], g["alphas"] = of3.backward(scene["scales"], scene["alphas"], filt, g["scales"], dalpha_f)
    if pose:
        per = camera_grad(st, scene["pws"], Rcw, cam["fx"], cam["fy"], W, H, du, dc, dcol, dz, model=model)["per"]
        if aa:
            per = per + camera_grad(oaa._identity_conic(st), scene["pws"], Rcw, cam["fx"], cam["fy"], W, H,
                                    np.zeros((N, 2)), gc2, np.zeros((N, 3)), model=model)["per"]
    else:
        per = np.zeros((N, 15))
    R64 = np.asarray(Rcw, np.float32).astype(np.float64).reshape(3, 3)
    pc64 = np.asarray(scene["pws"], np.float32).astype(np.float64) @ R64.T + np.asarray(cam["tcw"], np.float32)
    band = np.abs(pc64[:, 2] - 0.2) < ostep.Z_BAND
    band |= (pc64[:, 2] >= 0.2) & opencv_band(pc64, k, cam["fx"], cam["fy"], cam["cx"], cam["cy"], W, H)
    thin = oaa.thin(sf)
    flagged = amb | band | thin
    if aa:
        flagged = flagged | oaa.flagged(sf, s)
    return dict(image=out["image"], depth=out.get("depth"), alpha=out.get("alpha"), ambiguous=out["ambiguous"],
                grads=g, raster=(du, dc, da, dcol, dz), per=per, absum=np.abs(per).sum(0), cam_grad=per.sum(0),
                flagged=flagged, thin=thin, band=band, st=st, rho=rho, drawn=rho * af)
