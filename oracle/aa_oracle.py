"""fp64 antialiasing (2D-filter opacity compensation) of the per-Gaussian stages.  TEST
INFRASTRUCTURE ONLY.

With (a, b, c) the pre-blur cov2d, (a', b, c') = (a + w, b, c + w) the blurred one the oracle's
compute_cov2d returns (w = 0.3) and D = a' c' - b^2:
    r = (a c - b^2) / D,   rho = sqrt(max(2.5e-5, r)),   alpha_eff = rho alpha   (rho = 1 culled)
    dr/da = w (c c' + b^2) / D^2,  dr/db = -2 w b (w + a + c) / D^2,  dr/dc = w (a a' + b^2) / D^2
    drho = dr / (2 rho), 0 where the clamp holds (r <= 2.5e-5)
The addend alpha dL/dalpha_eff drho/d(a, b, c) to dL/dcov2d goes through the oracle's own
Jacobians (dcov2d_dcov3ds, dcov2d_dpcs) and, for the camera, pose_oracle.camera_grad.
"""
import numpy as np

from . import oracle as orc
from . import pose_oracle as opose

BLUR = 0.3
R_MIN = 2.5e-5


def stages(pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy, width, height):
    """pose_oracle.stages plus the blurred cov2d c2[N,3] (fp64, 0 for culled rows) the stages saw"""
    st = opose.stages(pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy, width, height)
    st["c2"] = orc.compute_cov2d(st["cov3ds"], st["pcs"], Rcw, st["depths"], fx, fy, width, height, calc_J=False)[0]
    return st


def scale(c2, keep):
    """-> dict(rho[N], r[N], kappa[N] (condition of the pre-blur determinant a c - b^2), clamped[N]
    (r <= R_MIN on a kept row), near[N] (r within a relative 1e-4 of R_MIN: the gradient jumps))"""
    c2 = np.asarray(c2, np.float64).reshape(-1, 3)
    keep = np.asarray(keep, bool).reshape(-1)
    a, b, c = c2[:, 0] - BLUR, c2[:, 1], c2[:, 2] - BLUR
    det = a * c - b * b
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(keep, det / (c2[:, 0] * c2[:, 2] - b * b), 1.0)
        kappa = np.where(keep, (np.abs(a * c) + b * b) / np.abs(det), 1.0)
    rho = np.where(keep, np.sqrt(np.maximum(R_MIN, r)), 1.0)
    return dict(rho=rho, r=r, kappa=kappa, clamped=keep & (r <= R_MIN),
                near=keep & (np.abs(r - R_MIN) <= 1e-4 * R_MIN))


def rel_tol(s):
    """relative tolerance of an fp32 rho against the oracle's (s: `scale`): r = (a c - b^2) / D loses kappa
    times the relative error of the fp32 cov2d entries (a few ulps: they come through cov3d and J), and
    rho = sqrt(r) halves it; 2^-19 kappa bounds the measured error with margin"""
    return 2e-5 + 2.0 ** -19 * np.nan_to_num(s["kappa"], nan=1.0)  # nan: a = b = c = 0 (clamped)


def thin(scales):
    """rows whose 3D covariance has thin axes fp32 cannot resolve next to its long one: the cov3d entries
    round at 2^-24 s_max^2, so whatever depends on the thin axes keeps few digits once s_max^2 / s_min^2
    nears 2^24 (r here; the conic and its gradients, and the pixels' exponent, on every path)"""
    sc3 = np.abs(np.asarray(scales, np.float64)).reshape(-1, 3)
    with np.errstate(divide="ignore", invalid="ignore"):
        k3d = np.nan_to_num((sc3.max(1) / sc3.min(1)) ** 2, nan=1.0, posinf=np.inf)
    return k3d > 1e4


def flagged(scales, s):
    """rows an fp32 AA gradient is bounded separately on: at the clamp, an ill-conditioned 2D determinant,
    or `thin`.  scales: those drawn."""
    return s["near"] | (rel_tol(s) > 1e-3) | thin(scales)


def dcov2d_addend(c2, keep, alphas, dloss_dalphas_eff):
    """alpha dL/dalpha_eff drho/d(a, b, c) -> [N,3] (0 on culled and clamped rows)"""
    c2 = np.asarray(c2, np.float64).reshape(-1, 3)
    s = scale(c2, keep)
    a1, b, c1 = c2[:, 0], c2[:, 1], c2[:, 2]
    a, c = a1 - BLUR, c1 - BLUR
    D = a1 * c1 - b * b
    live = np.asarray(keep, bool).reshape(-1) & ~s["clamped"]
    with np.errstate(divide="ignore", invalid="ignore"):
        k = np.where(live, np.asarray(alphas, np.float64).reshape(-1) *
                     np.asarray(dloss_dalphas_eff, np.float64).reshape(-1) * BLUR / (D * D) / (2.0 * s["rho"]), 0.0)
    g = np.stack([k * (c * c1 + b * b), k * (-2.0 * b * (BLUR + a + c)), k * (a * a1 + b * b)], axis=1)
    g[~live] = 0.0
    return g


def _identity_conic(st):
    """st with dconic/dcov2d replaced by I: a dL/dcov2d handed in as `dloss_dcinv2ds` then goes
    through the remaining Jacobians unchanged"""
    Ju, J3r, J3s, J2c, J2p, Jcs, Jcp, Jci = st["J"]
    out = dict(st)
    out["J"] = (Ju, J3r, J3s, J2c, J2p, Jcs, Jcp, np.broadcast_to(np.eye(3), Jci.shape).copy())
    return out


def chain(st, Rcw, gc2):
    """a dL/dcov2d addend gc2[N,3] through dcov2d_dcov3ds, dcov3d_d(rots, scales) and dcov2d_dpcs Rcw
    -> dict(pws[N,3], scales[N,3], rots[N,4])"""
    N = gc2.shape[0]
    z = lambda *s: np.zeros((N,) + s)
    ref = orc.chain_backward(Rcw, z(1, 2), gc2.reshape(N, 1, 3), z(1, 1), z(1, 3), *_identity_conic(st)["J"])
    return dict(pws=ref["pws"], scales=ref["scales"], rots=ref["rots"])


def camera(st, pws, Rcw, fx, fy, width, height, gc2):
    """the camera-gradient addend of gc2 (pose_oracle.camera_grad with dL/dcov2d given directly)
    -> per[N,15]"""
    N = gc2.shape[0]
    return opose.camera_grad(_identity_conic(st), pws, Rcw, fx, fy, width, height, np.zeros((N, 2)), gc2,
                             np.zeros((N, 3)))["per"]
