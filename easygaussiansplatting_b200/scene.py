"""Deterministic synthetic 3DGS scenes (SURVEY.md 8d / BASELINE.md 3).

There is no dataset on the GPU box, so every benchmark and full-size parity test renders a
seeded random scene of the shape BASELINE.json names.  numpy only; the arrays follow the
reference's Gaussian record (gsplat/gau_io.py:7-12: pw[3], rot[4] (w,x,y,z), scale[3],
alpha, sh[sh_dim] laid out [coef][rgb]) and its Camera fields
(gsplat/gausplat_dataset.py:14-27).
"""
import math

import numpy as np


def synthetic_scene(N, width, height, sh_dim=48, seed=0):
    """camera Rcw=I, tcw=0, fx=fy=W/(2 tan30deg), cx=W/2, cy=H/2.  Per Gaussian:
    z~U(2,12); target pixel u~U(-0.05W,1.05W), v~U(-0.05H,1.05H); pw back-projected;
    per-axis pixel sigma ~ LogU(0.5,4) -> scale = sigma*z/fx; rot = normalised N(0,1)^4;
    alpha~U(0.05,0.95); sh[:, :3]~N(0,1), higher bands ~N(0,0.2^2)."""
    rng = np.random.default_rng(seed)
    W, H = int(width), int(height)
    fx = fy = W / (2.0 * math.tan(math.radians(30.0)))
    cx, cy = W / 2.0, H / 2.0
    z = rng.uniform(2.0, 12.0, N)
    u = rng.uniform(-0.05 * W, 1.05 * W, N)
    v = rng.uniform(-0.05 * H, 1.05 * H, N)
    pws = np.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], axis=1)
    sig = np.exp(rng.uniform(math.log(0.5), math.log(4.0), (N, 3)))
    scales = sig * z[:, None] / fx
    rots = rng.normal(size=(N, 4))
    rots /= np.linalg.norm(rots, axis=1, keepdims=True)
    alphas = rng.uniform(0.05, 0.95, N)
    shs = rng.normal(size=(N, sh_dim))
    shs[:, 3:] *= 0.2
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    return dict(pws=f32(pws), rots=f32(rots), scales=f32(scales), alphas=f32(alphas),
                shs=f32(shs), Rcw=np.eye(3, dtype=np.float32), tcw=np.zeros(3, np.float32),
                twc=np.zeros(3, np.float32), fx=float(fx), fy=float(fy), cx=float(cx),
                cy=float(cy), width=W, height=H)


def upstream_gradient(width, height, seed=0):
    """dloss_dgammas ~ N(0,1)/(3WH), planar [3,H,W] float32 (SURVEY 8d)."""
    rng = np.random.default_rng(seed + 1000003)
    g = rng.normal(size=(3, int(height), int(width))) / (3.0 * width * height)
    return np.ascontiguousarray(g, dtype=np.float32)


def ring_camera(k, n_views, radius=0.6):
    """View k of n on a small ring around the synthetic camera (config 5: one camera per
    rank over shared Gaussians).  Returns Rcw, tcw, twc float32."""
    a = 2.0 * math.pi * k / max(1, n_views)
    yaw = 0.05 * math.sin(a)
    c, s = math.cos(yaw), math.sin(yaw)
    Rcw = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]], dtype=np.float64)
    twc = np.array([radius * math.cos(a), radius * math.sin(a) * 0.5, 0.0])
    tcw = -Rcw @ twc
    return Rcw.astype(np.float32), tcw.astype(np.float32), twc.astype(np.float32)


COLMAP_LIKE_FISHEYE_K = (0.05, -0.01, 0.002, -0.0005)  # k1..k4 of a typical OPENCV_FISHEYE calibration
# (k1, k2), (p1, p2) of a typical OPENCV calibration of a moderately wide lens
COLMAP_LIKE_OPENCV = ((-0.12, 0.03), (4e-4, -6e-4))


def opencv_undistort(mx, my, k, iters=20):
    """(xn, yn) with delta(xn, yn) = (mx, my) for the opencv lens k = (k1, k2, p1, p2) (ops.preprocess).
    The radial part is solved first by bisection on [0, r_max), where r (1 + k1 r^2 + k2 r^4) increases;
    Newton steps on delta then add the tangential part.  A target beyond the radial curve's maximum
    lands at 1.02 r_max on its ray: past the fold, where the kernels cull."""
    k1, k2, p1, p2 = (float(v) for v in k)
    mx, my = np.asarray(mx, np.float64), np.asarray(my, np.float64)
    rd = np.hypot(mx, my)
    # r_max^2: the smallest positive root of 1 + 3 k1 rho + 5 k2 rho^2
    roots = np.roots([5 * k2, 3 * k1, 1.0]) if k2 != 0 else ([-1 / (3 * k1)] if k1 != 0 else [])
    pos = [r.real for r in np.atleast_1d(roots) if abs(np.imag(r)) < 1e-12 and r.real > 0]
    rmax = math.sqrt(min(pos)) if pos else math.inf
    dist = lambda r: r * (1 + r * r * (k1 + r * r * k2))
    lo = np.zeros_like(rd)
    if math.isfinite(rmax):
        hi = np.full_like(rd, rmax)
        beyond = dist(hi) < rd
    else:
        hi = np.maximum(2 * rd, 1.0)
        while (dist(hi) < rd).any():
            hi = np.where(dist(hi) < rd, 2 * hi, hi)
        beyond = np.zeros(rd.shape, bool)
    for _ in range(80):
        m = 0.5 * (lo + hi)
        below = dist(m) < rd
        lo, hi = np.where(below, m, lo), np.where(below, hi, m)
    ru = np.where(beyond, 1.02 * rmax if math.isfinite(rmax) else 0.0, 0.5 * (lo + hi))
    with np.errstate(invalid="ignore", divide="ignore"):
        s = np.where(rd > 0, ru / rd, 1.0)
    x, y = mx * s, my * s
    for _ in range(iters):
        rho = x * x + y * y
        R, R1 = 1 + rho * (k1 + rho * k2), k1 + 2 * k2 * rho
        ex = x * R + 2 * p1 * x * y + p2 * (rho + 2 * x * x) - mx
        ey = y * R + p1 * (rho + 2 * y * y) + 2 * p2 * x * y - my
        d00 = R + 2 * x * x * R1 + 2 * p1 * y + 6 * p2 * x
        d01 = 2 * x * y * R1 + 2 * p1 * x + 2 * p2 * y
        d11 = R + 2 * y * y * R1 + 6 * p1 * y + 2 * p2 * x
        det = d00 * d11 - d01 * d01
        with np.errstate(invalid="ignore", divide="ignore"):
            nx, ny = x - (d11 * ex - d01 * ey) / det, y - (d00 * ey - d01 * ex) / det
        x, y = np.where(beyond, x, nx), np.where(beyond, y, ny)
    return x, y


def camera_model_scene(N, width, height, camera_model="pinhole", radial_coeffs=None, sh_dim=48, seed=0,
                       tangential_coeffs=None):
    """synthetic_scene with its target pixels unprojected through a camera model instead of the pinhole,
    so that scenes of different models cover the frame alike.  pinhole: synthetic_scene itself.
    ortho: fx = fy = W / 16 (16 world units across); pw = ((u - cx) / fx, (v - cy) / fy, z).
    fisheye (Kannala-Brandt k1..k4 = radial_coeffs, default 0): fx = fy = W / pi, 180 degrees across the
    width; the pixel's ray (theta_d -> theta by Newton) at distance z.  Targets beyond theta = 90 degrees (the
    corners) land behind the camera and are culled.
    opencv (k1, k2 = radial_coeffs, p1, p2 = tangential_coeffs, default 0): synthetic_scene's fx, fy;
    the pixel's undistorted point (`opencv_undistort`) at depth z.
    Scales: the pixel sigma times the metres per pixel at the Gaussian (z / fx; 1 / fx for ortho).
    -> the dict of synthetic_scene plus camera_model, radial_coeffs, tangential_coeffs"""
    sc = synthetic_scene(N, width, height, sh_dim=sh_dim, seed=seed)
    sc["camera_model"], sc["radial_coeffs"] = camera_model, radial_coeffs
    sc["tangential_coeffs"] = tangential_coeffs
    if camera_model == "pinhole":
        return sc
    rng = np.random.default_rng(seed)  # the same draws as synthetic_scene
    W, H = int(width), int(height)
    cx, cy = W / 2.0, H / 2.0
    z = rng.uniform(2.0, 12.0, N)
    u = rng.uniform(-0.05 * W, 1.05 * W, N)
    v = rng.uniform(-0.05 * H, 1.05 * H, N)
    sig = np.exp(rng.uniform(math.log(0.5), math.log(4.0), (N, 3)))
    if camera_model == "ortho":
        f = W / 16.0
        pws = np.stack([(u - cx) / f, (v - cy) / f, z], axis=1)
        scales = sig / f
    elif camera_model == "fisheye":
        f = W / math.pi
        k1, k2, k3, k4 = radial_coeffs if radial_coeffs is not None else (0.0, 0.0, 0.0, 0.0)
        mx, my = (u - cx) / f, (v - cy) / f
        td = np.hypot(mx, my)
        th = td.copy()
        for _ in range(30):
            t2 = th * th
            fth = th * (1 + t2 * (k1 + t2 * (k2 + t2 * (k3 + t2 * k4)))) - td
            th -= fth / (1 + t2 * (3 * k1 + t2 * (5 * k2 + t2 * (7 * k3 + t2 * 9 * k4))))
        phi = np.arctan2(my, mx)
        pws = np.stack([z * np.sin(th) * np.cos(phi), z * np.sin(th) * np.sin(phi), z * np.cos(th)], axis=1)
        scales = sig * z[:, None] / f
    elif camera_model == "opencv":
        f = sc["fx"]
        k = tuple(radial_coeffs or (0.0, 0.0)) + tuple(tangential_coeffs or (0.0, 0.0))
        xn, yn = opencv_undistort((u - cx) / f, (v - cy) / f, k)
        pws = np.stack([xn * z, yn * z, z], axis=1)
        scales = sig * z[:, None] / f
    else:
        raise ValueError("unknown camera model %r" % (camera_model,))
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    sc.update(pws=f32(pws), scales=f32(scales), fx=float(f), fy=float(f))
    return sc
