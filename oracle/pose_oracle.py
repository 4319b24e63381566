"""fp64 camera gradient of the per-Gaussian stages.  TEST INFRASTRUCTURE ONLY.

dL/dRcw, dL/dtcw, dL/dtwc summed over the Gaussians, built from the oracle's own per-Gaussian
Jacobians (oracle.project / compute_cov2d / sh2color / inverse_cov2d, which the reference's
code pins), with pc = Rcw pw + tcw and M = J Rcw:
    dL/dpc  = dL/du du/dpc + dL/dcov2d dcov2d/dpc (+ dL/dz on pc[2])    (kept Gaussians only)
    dL/dtcw = sum dL/dpc
    dL/dRcw = sum dL/dpc (x) pw + J^T dL/dM          (dL/dM = 2 G M Sigma, the direct use of Rcw)
    dL/dtwc = -sum dL/dcolor dcolor/dpw               (the view direction is pw - twc)
The only new derivative is the direct term, evaluated here in fp64 from the cov3ds and pcs
compute_cov2d was given; J uses the clamped x, y exactly as compute_cov2d does.
"""
import numpy as np

from . import oracle as orc


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def stages(pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy, width, height):
    """The five oracle stages with Jacobians, as the chain tests run them.  -> dict(us, ci, col,
    depths (f32, after the NaN-determinant cull; < 0 = culled), areas, keep[N] bool, pcs and
    cov3ds (the fp32 values compute_cov2d read), J = chain_backward's eight Jacobians)"""
    us, pcs, depths, Ju = orc.project(pws, Rcw, tcw, fx, fy, cx, cy)
    d32 = _f32(depths)
    c3, J3r, J3s = orc.compute_cov3d(rots, scales, d32)
    c3, pcs = _f32(c3), _f32(pcs)
    c2, J2c, J2p = orc.compute_cov2d(c3, pcs, Rcw, d32, fx, fy, width, height)
    col, Jcs, Jcp = orc.sh2color(shs, pws, twc)
    ci, areas, Jci = orc.inverse_cov2d(_f32(c2), d32)
    return dict(us=us, ci=ci, col=col, depths=d32, areas=areas, keep=d32 >= 0.2, pcs=pcs, cov3ds=c3,
                J=(Ju, J3r, J3s, J2c, J2p, Jcs, Jcp, Jci))


def camera_grad(st, pws, Rcw, fx, fy, width, height, dloss_dus, dloss_dcinv2ds, dloss_dcolors,
                dloss_ddepths=None):
    """The camera gradient from `stages` output st and the four upstream gradients ([N,2], [N,3],
    [N,3], [N] or None).  -> dict(grad[15] = dL/dRcw (row-major 9), dL/dtcw (3), dL/dtwc (3);
    per[N,15] the Gaussians' contributions; absum[15] = sum_i |per_i|, the scale tolerances use)"""
    f = lambda a: np.asarray(a, dtype=np.float64)
    Ju, _, _, _, J2p, _, Jcp, Jci = (f(a) for a in st["J"])
    N = Ju.shape[0]
    R = f(_f32(Rcw)).reshape(3, 3)
    pw = f(_f32(pws)).reshape(N, 3)
    gu = f(dloss_dus).reshape(N, 2)
    gci = f(dloss_dcinv2ds).reshape(N, 3)
    gcol = f(dloss_dcolors).reshape(N, 3)
    keep = np.asarray(st["keep"], bool).reshape(N)
    gc2 = np.einsum("ni,nij->nj", gci, Jci)                      # dL/dcov2d (a, b, c)
    gpc = np.einsum("ni,nij->nj", gu, Ju) + np.einsum("ni,nij->nj", gc2, J2p)
    if dloss_ddepths is not None:
        gpc[:, 2] += f(dloss_ddepths).reshape(N)
    gpc[~keep] = 0.0
    # direct term: cov2d = M Sigma M^T + 0.3 I, M = J Rcw  ->  dL/dRcw += J^T (2 G M Sigma)
    pc = f(st["pcs"]).reshape(N, 3)
    c3 = f(st["cov3ds"]).reshape(N, 6)
    z = np.where(keep, pc[:, 2], 1.0)
    limx = 1.3 * (float(width) / (2.0 * np.float32(fx)))
    limy = 1.3 * (float(height) / (2.0 * np.float32(fy)))
    xc = np.clip(pc[:, 0] / z, -limx, limx) * z
    yc = np.clip(pc[:, 1] / z, -limy, limy) * z
    fx, fy = float(np.float32(fx)), float(np.float32(fy))
    J = np.zeros((N, 2, 3))
    J[:, 0, 0] = fx / z; J[:, 0, 2] = -fx * xc / z ** 2
    J[:, 1, 1] = fy / z; J[:, 1, 2] = -fy * yc / z ** 2
    S = c3[:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(N, 3, 3)
    G = np.stack([gc2[:, 0], 0.5 * gc2[:, 1], 0.5 * gc2[:, 1], gc2[:, 2]], axis=1).reshape(N, 2, 2)
    M = J @ R[None]
    dM = 2.0 * G @ M @ S
    dR = np.einsum("nai,naj->nij", J, dM)
    dR[~keep] = 0.0
    per = np.zeros((N, 15))
    per[:, :9] = (gpc[:, :, None] * pw[:, None, :] + dR).reshape(N, 9)
    per[:, 9:12] = gpc
    per[:, 12:15] = -np.einsum("nc,ncb->nb", gcol, Jcp)          # colour branch: not gated by depth
    return dict(grad=per.sum(0), per=per, absum=np.abs(per).sum(0))


def chain_twc(grad, Rcw, tcw):
    """The raw gradient chained through twc = -Rcw^T tcw (what autograd delivers to Rcw and tcw when
    the caller builds twc that way).  -> (dRcw[3,3], dtcw[3])"""
    g = np.asarray(grad, dtype=np.float64)
    R = np.asarray(Rcw, dtype=np.float64).reshape(3, 3)
    t = np.asarray(tcw, dtype=np.float64).reshape(3)
    dR, dt, dw = g[:9].reshape(3, 3), g[9:12], g[12:15]
    # twc[k] = -sum_j R[j,k] t[j]:  dtwc/dR[j,k] = -t[j],  dtwc/dt[j] = -R[j,:]
    return dR - np.outer(t, dw), dt - R @ dw
