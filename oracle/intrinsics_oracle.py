"""fp64 intrinsics gradient of the per-Gaussian stages (DESIGN 3.23).  TEST INFRASTRUCTURE ONLY.

Per kept Gaussian, with theta = (fx, fy, cx, cy, k[4]) (k: opencv's k1, k2, p1, p2, fisheye's k1..k4,
unused by pinhole and ortho), the projected mean u(theta) and the EWA Jacobian J(theta):
    dL/dtheta = dL/du . du/dtheta + sum_ab dL/dJ_ab dJ_ab/dtheta,   dL/dJ = 2 G J (R Sigma R^T)
with G = sym(dL/dcov2d) and dL/dcov2d = dL/dconic . dconic/dcov2d (+ antialiasing's alpha dL/dalpha_eff
drho/dcov2d, aa_oracle.dcov2d_addend).  The clamp bound lim = (Lx, Ly) (pinhole: 1.3 tan_fov; opencv:
opencv_oracle.opencv_limits) is a constant: a clamped coordinate enters J at the bound, and nothing
differentiates the bound.  `forward` evaluates u, the conic and rho at given intrinsics with the bound
pinned, so central differences of it check `per_gaussian`.  `step` is opencv_oracle.step (every model)
with the intrinsics gradient of the same upstream gradients added.
"""
import numpy as np

from . import aa_oracle as oaa
from . import camera_model_oracle as ocm
from . import opencv_oracle as ocv

MODELS = ("pinhole", "ortho", "fisheye", "opencv")


def limits(model, intr, width, height):
    """the constant clamp bound (Lx, Ly) of a camera, from its fp32 intrinsics (None: no clamp)"""
    fx, fy, cx, cy = (float(np.float32(v)) for v in intr[:4])
    if model == "pinhole":
        return 1.3 * width / (2 * fx), 1.3 * height / (2 * fy)
    if model == "opencv":
        return ocv.opencv_limits(np.asarray(intr[4:], np.float64), fx, fy, cx, cy, float(width), float(height))
    return None


def dproj(pc, model, intr, lim=None):
    """-> u[N,2], J[N,2,3], du[N,2,8] = du/dtheta, dJ[N,2,3,8] = dJ/dtheta at pc[N,3] (fp64)"""
    pc = np.asarray(pc, np.float64).reshape(-1, 3)
    N = len(pc)
    x, y, z = pc[:, 0], pc[:, 1], pc[:, 2]
    fx, fy, cx, cy = (float(v) for v in intr[:4])
    k = np.asarray(intr[4:], np.float64)
    f = (fx, fy)
    du, dJ = np.zeros((N, 2, 8)), np.zeros((N, 2, 3, 8))
    du[:, 0, 2] = du[:, 1, 3] = 1.0
    if model in ("pinhole", "ortho"):
        if model == "pinhole":
            a, b = x / z, y / z
            ah, bh = np.clip(a, -lim[0], lim[0]), np.clip(b, -lim[1], lim[1])
            F = np.zeros((N, 2, 3))  # J / diag(f)
            F[:, 0, 0], F[:, 0, 2], F[:, 1, 1], F[:, 1, 2] = 1 / z, -ah / z, 1 / z, -bh / z
            m = np.stack([a, b], 1)
        else:
            F = np.zeros((N, 2, 3))
            F[:, 0, 0] = F[:, 1, 1] = 1.0
            m = np.stack([x, y], 1)
    elif model == "fisheye":
        T = ocm.fisheye_terms(pc, k)
        s, g, h, th = T["s"], T["g"], T["h"], T["theta"]
        r2 = x * x + y * y
        q, t = r2 + z * z, np.sqrt(r2) / z
        with np.errstate(divide="ignore", invalid="ignore"):
            tht = np.where(t < 1e-3, 1 - t * t / 3 + t ** 4 / 5, th / t)  # theta / t
        xy = (x, y)
        F = np.zeros((N, 2, 3))
        for a_ in range(2):
            for b_ in range(2):
                F[:, a_, b_] = (s if a_ == b_ else 0.0) + xy[a_] * xy[b_] * g
            F[:, a_, 2] = -xy[a_] * h
        m = np.stack([s * x, s * y], 1)
        for j in range(4):
            p, c = th ** (2 * j + 2), 2 * j + 3
            ds = p * tht / z                                        # theta^(2j+3) / r
            dg = (tht / z) ** 2 * th ** (2 * j) * (c * z / q - tht / z)  # ((c theta^2j+2 z/q - ds) / r^2
            dh = c * p / q
            for a_ in range(2):
                du[:, a_, 4 + j] = f[a_] * xy[a_] * ds
                for b_ in range(2):
                    dJ[:, a_, b_, 4 + j] = f[a_] * ((ds if a_ == b_ else 0.0) + xy[a_] * xy[b_] * dg)
                dJ[:, a_, 2, 4 + j] = -f[a_] * xy[a_] * dh
    elif model == "opencv":
        a, b = x / z, y / z
        ah, bh = np.clip(a, -lim[0], lim[0]), np.clip(b, -lim[1], lim[1])
        dlt = ocv.opencv_terms(a, b, k)[0]
        D = ocv.opencv_terms(ah, bh, k)[1]
        F = np.zeros((N, 2, 3))
        for r_, (d0, d1) in ((0, (D[0], D[1])), (1, (D[1], D[2]))):
            F[:, r_, 0], F[:, r_, 1], F[:, r_, 2] = d0 / z, d1 / z, -(d0 * ah + d1 * bh) / z
        m = np.stack(dlt, 1)
        ru, rc = a * a + b * b, ah * ah + bh * bh
        # d delta / d(k1, k2, p1, p2) at (a, b); d Ddelta (00, 01, 11) / d(...) at (ah, bh)
        ddl = ((a * ru, b * ru), (a * ru * ru, b * ru * ru), (2 * a * b, ru + 2 * b * b), (ru + 2 * a * a, 2 * a * b))
        dD = ((rc + 2 * ah * ah, 2 * ah * bh, rc + 2 * bh * bh),
              (rc * (rc + 4 * ah * ah), 4 * ah * bh * rc, rc * (rc + 4 * bh * bh)),
              (2 * bh, 2 * ah, 6 * bh), (6 * ah, 2 * bh, 2 * ah))
        for j in range(4):
            for r_, (i0, i1) in ((0, (0, 1)), (1, (1, 2))):
                du[:, r_, 4 + j] = f[r_] * ddl[j][r_]
                e0, e1 = dD[j][i0], dD[j][i1]
                dJ[:, r_, 0, 4 + j] = f[r_] * e0 / z
                dJ[:, r_, 1, 4 + j] = f[r_] * e1 / z
                dJ[:, r_, 2, 4 + j] = -f[r_] * (e0 * ah + e1 * bh) / z
    else:
        raise ValueError("unknown camera model %r" % (model,))
    u = np.stack([fx * m[:, 0] + cx, fy * m[:, 1] + cy], 1)
    J = F * np.array([fx, fy])[None, :, None]
    du[:, 0, 0], du[:, 1, 1] = m[:, 0], m[:, 1]
    dJ[:, 0, :, 0], dJ[:, 1, :, 1] = F[:, 0], F[:, 1]
    return u, J, du, dJ


def _cov2d(J, R, c3):
    S = np.asarray(c3, np.float64).reshape(-1, 6)[:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(-1, 3, 3)
    Sp = R[None] @ S @ R.T[None]
    C = J @ Sp @ J.transpose(0, 2, 1)
    return np.stack([C[:, 0, 0] + oaa.BLUR, C[:, 0, 1], C[:, 1, 1] + oaa.BLUR], 1), Sp


def forward(pc, R, cov3d, model, intr, lim):
    """-> u[N,2], conic[N,3], rho[N] (antialiasing's opacity scale, unclamped) with the bound pinned"""
    u, J, _, _ = dproj(pc, model, intr, lim)
    c2, _ = _cov2d(J, np.asarray(R, np.float64).reshape(3, 3), cov3d)
    a, b, c = c2[:, 0], c2[:, 1], c2[:, 2]
    det = a * c - b * b
    rho = np.sqrt(np.maximum((a - oaa.BLUR) * (c - oaa.BLUR) - b * b, 0.0) / det)
    return u, np.stack([c / det, -b / det, a / det], 1), rho


def per_gaussian(pc, R, cov3d, model, intr, lim, gu, gconic, gc2_add=None, keep=None, magnitude=False):
    """the Gaussians' contributions [N,8] to dL/dtheta from dL/du gu[N,2], dL/dconic gconic[N,3] and an
    optional dL/dcov2d addend gc2_add[N,3]; rows where keep is False contribute 0.  magnitude: also the
    sum of the absolute values of each contribution's terms [N,8] (|gu_a du_a/dtheta| and |dL/dJ_ab
    dJ_ab/dtheta|), the scale an fp32 evaluation of the same sum is held to"""
    R = np.asarray(R, np.float64).reshape(3, 3)
    _, J, du, dJt = dproj(pc, model, intr, lim)
    c2, Sp = _cov2d(J, R, cov3d)
    a, b, c = c2[:, 0], c2[:, 1], c2[:, 2]
    di = 1.0 / (a * c - b * b)
    d2 = di * di
    g = np.asarray(gconic, np.float64).reshape(-1, 3)
    ga = g[:, 0] * (-c * c * d2) + g[:, 1] * (b * c * d2) + g[:, 2] * (di - a * c * d2)
    gb = g[:, 0] * (2 * b * c * d2) + g[:, 1] * (-di - 2 * b * b * d2) + g[:, 2] * (2 * a * b * d2)
    gc = g[:, 0] * (di - a * c * d2) + g[:, 1] * (a * b * d2) + g[:, 2] * (-a * a * d2)
    if gc2_add is not None:
        ga, gb, gc = ga + gc2_add[:, 0], gb + gc2_add[:, 1], gc + gc2_add[:, 2]
    G = np.stack([ga, 0.5 * gb, 0.5 * gb, gc], 1).reshape(-1, 2, 2)
    dLdJ = 2.0 * G @ J @ Sp
    per = np.einsum("na,nat->nt", np.asarray(gu, np.float64).reshape(-1, 2), du) + np.einsum("nab,nabt->nt", dLdJ, dJt)
    mag = np.einsum("na,nat->nt", np.abs(np.asarray(gu, np.float64).reshape(-1, 2)), np.abs(du)) + \
        np.einsum("nab,nabt->nt", np.abs(dLdJ), np.abs(dJt))
    if keep is not None:
        per[~np.asarray(keep, bool)] = 0.0
        mag[~np.asarray(keep, bool)] = 0.0
    return (per, mag) if magnitude else per


def kernel_upstream(moments, cinv2ds):
    """dL/du, dL/dconic, dL/dalpha_eff exactly as the fused backward reads them from fp32 moment rows and
    conics, in fp64"""
    m = np.asarray(moments, np.float64).reshape(-1, 9)
    ci = np.asarray(cinv2ds, np.float64).reshape(-1, 3)
    none = (m[:, 0] == 0) & (m[:, 1] == 0)
    gu = -np.stack([ci[:, 0] * m[:, 0] + ci[:, 1] * m[:, 1], ci[:, 1] * m[:, 0] + ci[:, 2] * m[:, 1]], 1)
    gu[none] = 0.0
    return gu, np.stack([-0.5 * m[:, 2], -m[:, 3], -0.5 * m[:, 4]], 1), m[:, 5]


def step(scene, cam, *, rgbd, aa, filt, dl, dld=None, dla=None, model="pinhole", k=None):
    """opencv_oracle.step with pose=True plus the intrinsics gradient: 'iper'[N,8], 'intr_grad'[8] and
    'iabsum'[8] (sum of |contribution|) from the same rasterizer gradients (antialiasing's term included)"""
    out = ocv.step(scene, cam, rgbd=rgbd, pose=True, aa=aa, filt=filt, dl=dl, dld=dld, dla=dla, model=model, k=k)
    if "st" not in out:  # pinhole: step_oracle.step keeps the stages in its forward's dict
        out.update(st=out["fwd"]["st"], rho=out["fwd"]["rho"], drawn=out["fwd"]["drawn"])
    st = out["st"]
    du, dc, da, _, _ = out["raster"]
    kk = np.zeros(4) if k is None else np.asarray(k, np.float64)
    intr = [float(np.float32(cam[n])) for n in ("fx", "fy", "cx", "cy")] + [float(np.float32(v)) for v in kk]
    lim = limits(model, intr, cam["width"], cam["height"])
    N = len(st["keep"])
    keep = np.asarray(st["keep"], bool)
    pc = np.where(keep[:, None], np.asarray(st["pcs"], np.float64), [0.0, 0.0, 1.0])
    af = np.asarray(out["drawn"], np.float64) / out["rho"]
    gc2 = oaa.dcov2d_addend(st["c2"], keep, af, np.asarray(da, np.float64).reshape(N)) if aa else None
    per = per_gaussian(pc, cam["Rcw"], st["cov3ds"], model, intr, lim, np.asarray(du).reshape(N, 2), dc, gc2,
                       keep)
    out.update(iper=per, intr_grad=per.sum(0), iabsum=np.abs(per).sum(0))
    return out
