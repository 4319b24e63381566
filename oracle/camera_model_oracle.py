"""fp64 camera models (pinhole, ortho, fisheye) of the per-Gaussian stages.  TEST INFRASTRUCTURE ONLY.

Per model, at a camera-frame point pc = (x, y, z):
    pinhole  u = (fx x/z + cx, fy y/z + cy)                           (no fov clamp here)
    ortho    u = (fx x + cx, fy y + cy)
    fisheye  theta = atan2(r, z), r = |(x, y)|, theta_d = theta (1 + k1 theta^2 + ... + k4 theta^8),
             u = (fx theta_d x / r + cx, fy theta_d y / r + cy)         (Kannala-Brandt)
`project` returns u, J = du/dpc and dJ/dpc, from closed forms (DESIGN 3.14) in fp64; near the axis
(t = r/z < 1e-3, where the closed forms are 0/0) from their series in t^2.  The tests hold all three
against central differences.

`stages` builds the dict of pose_oracle.stages (the same keys and Jacobians, so oracle.chain_backward,
aa_oracle, rgbd_oracle.chain_depth and the rasterizer oracles compose with it) for any model: du_dpcs,
cov2d, dcov2d_dcov3ds and dcov2d_dpcs come from the model's J; cov3d, colour and the conic from the C
oracle.  The pinhole model is exactly pose_oracle.stages (the C oracle's clamped J).  `camera_grad`
and `step` are pose_oracle.camera_grad and step_oracle.step with the model's J in the direct term.
"""
import numpy as np

from . import aa_oracle as oaa
from . import filter3d_oracle as of3
from . import oracle as orc
from . import pose_oracle as opose
from . import rgbd_oracle as ordb
from . import step_oracle as ostep

MODELS = ("pinhole", "ortho", "fisheye")
SERIES_T = 1e-3


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _k(k):
    return np.zeros(4) if k is None else np.asarray(k, np.float64).reshape(4)


def fisheye_terms(pc, k=None):
    """-> dict(s, g, h, G, H, hz, P1 (theta_d'), theta) of the fisheye at pc[N,3] (fp64):
    u = f s (x, y),  g = (1/r) ds/dr,  h = -ds/dz,  G = (1/r) dg/dr,  H = (1/r) dh/dr = -dg/dz,  hz = dh/dz"""
    pc = np.asarray(pc, np.float64).reshape(-1, 3)
    k1, k2, k3, k4 = _k(k)
    x, y, z = pc[:, 0], pc[:, 1], pc[:, 2]
    r2 = x * x + y * y
    r, q = np.sqrt(r2), r2 + z * z
    t = r / z
    th = np.arctan2(r, z)
    th2 = th * th
    P = 1 + th2 * (k1 + th2 * (k2 + th2 * (k3 + th2 * k4)))
    P1 = 1 + th2 * (3 * k1 + th2 * (5 * k2 + th2 * (7 * k3 + th2 * 9 * k4)))
    P2 = 6 * k1 + th2 * (20 * k2 + th2 * (42 * k3 + th2 * 72 * k4))
    small = t < SERIES_T
    t2 = t * t
    a1, a2 = k1 - 1.0 / 3.0, 0.2 - k1 + k2
    with np.errstate(divide="ignore", invalid="ignore"):
        tht = np.where(small, 1 - t2 / 3 + t2 * t2 / 5, th / t)
        s = np.where(small, (1 + a1 * t2 + a2 * t2 * t2) / z, P * th / r)
        g = np.where(small, (2 * a1 + 4 * a2 * t2) / z ** 3, (P1 * z / q - P * th / r) / r2)
        A, sn2 = r * z / q, r2 / q
        F = P1 * A - P * th
        Fp = P2 * th * A - 2 * P1 * sn2
        G = np.where(small, 8 * a2 / z ** 5, (A * Fp - 3 * F) / (r2 * r2 * r))
    h = P1 / q
    H = (P2 * tht - 2 * P1) / (q * q)
    hz = -(P2 * th * r + 2 * z * P1) / (q * q)
    return dict(s=s, g=g, h=h, G=G, H=H, hz=hz, P1=P1, theta=th)


def project(pc, model, fx, fy, cx, cy, k=None):
    """-> u[N,2], J[N,2,3] = du/dpc, dJ[N,2,3,3] = dJ[a,b]/dpc[c], valid[N] (fisheye: theta_d' > 0)"""
    pc = np.asarray(pc, np.float64).reshape(-1, 3)
    N = pc.shape[0]
    x, y, z = pc[:, 0], pc[:, 1], pc[:, 2]
    fx, fy, cx, cy = (float(v) for v in (fx, fy, cx, cy))
    u = np.zeros((N, 2)); J = np.zeros((N, 2, 3)); dJ = np.zeros((N, 2, 3, 3))
    valid = np.ones(N, bool)
    if model == "pinhole":
        u[:, 0], u[:, 1] = fx * x / z + cx, fy * y / z + cy
        J[:, 0, 0], J[:, 0, 2] = fx / z, -fx * x / z ** 2
        J[:, 1, 1], J[:, 1, 2] = fy / z, -fy * y / z ** 2
        dJ[:, 0, 0, 2] = -fx / z ** 2
        dJ[:, 0, 2, 0], dJ[:, 0, 2, 2] = -fx / z ** 2, 2 * fx * x / z ** 3
        dJ[:, 1, 1, 2] = -fy / z ** 2
        dJ[:, 1, 2, 1], dJ[:, 1, 2, 2] = -fy / z ** 2, 2 * fy * y / z ** 3
    elif model == "ortho":
        u[:, 0], u[:, 1] = fx * x + cx, fy * y + cy
        J[:, 0, 0], J[:, 1, 1] = fx, fy
    elif model == "fisheye":
        T = fisheye_terms(pc, k)
        s, g, h, G, H, hz = (T[n] for n in ("s", "g", "h", "G", "H", "hz"))
        valid = T["P1"] > 0
        u[:, 0], u[:, 1] = fx * s * x + cx, fy * s * y + cy
        f = np.array([fx, fy])
        xy = (x, y)
        for a in range(2):
            ca = xy[a]
            # row a: J[a, b] = f_a (s delta_ab + c_a c_b g) for b < 2,  J[a, 2] = -f_a c_a h
            for b in range(2):
                J[:, a, b] = f[a] * ((s if a == b else 0.0) + ca * xy[b] * g)
            J[:, a, 2] = -f[a] * ca * h
            # ds/dc = c g, dg/dc = c G, dh/dc = c H (c = x, y);  ds/dz = -h, dg/dz = -H, dh/dz = hz
            for b in range(2):
                cb = xy[b]
                for c in range(2):
                    cc = xy[c]
                    d_cacb = (ca if b == c else 0.0) + (cb if a == c else 0.0)
                    dJ[:, a, b, c] = f[a] * ((cc * g if a == b else 0.0) + d_cacb * g + ca * cb * cc * G)
                dJ[:, a, b, 2] = f[a] * (-(h if a == b else 0.0) - ca * cb * H)
            for c in range(2):
                dJ[:, a, 2, c] = -f[a] * ((h if a == c else 0.0) + ca * xy[c] * H)
            dJ[:, a, 2, 2] = -f[a] * ca * hz
    else:
        raise ValueError("unknown camera model %r" % (model,))
    return u, J, dJ, valid


def unproject_fisheye(u, fx, fy, cx, cy, k=None, iters=50):
    """the unit ray of a fisheye pixel: theta_d = |((u - cx) / fx, (v - cy) / fy)|, theta_d(theta) solved by
    Newton from theta = theta_d -> dirs[N,3]"""
    u = np.asarray(u, np.float64).reshape(-1, 2)
    k1, k2, k3, k4 = _k(k)
    mx, my = (u[:, 0] - cx) / fx, (u[:, 1] - cy) / fy
    td = np.hypot(mx, my)
    th = td.copy()
    for _ in range(iters):
        t2 = th * th
        f = th * (1 + t2 * (k1 + t2 * (k2 + t2 * (k3 + t2 * k4)))) - td
        d = 1 + t2 * (3 * k1 + t2 * (5 * k2 + t2 * (7 * k3 + t2 * 9 * k4)))
        th = th - f / d
    with np.errstate(divide="ignore", invalid="ignore"):
        cphi = np.where(td > 0, mx / td, 1.0)
        sphi = np.where(td > 0, my / td, 0.0)
    return np.stack([np.sin(th) * cphi, np.sin(th) * sphi, np.cos(th)], axis=1)


def _cov2d(J, R, c3):
    """cov2d (a, b, c) + 0.3, dcov2d/dcov3d [N,3,6] and dcov2d/dpc needs of M = J R, Sigma"""
    N = J.shape[0]
    S = c3[:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(N, 3, 3)
    M = J @ R[None]
    C = M @ S @ M.transpose(0, 2, 1)
    c2 = np.stack([C[:, 0, 0] + oaa.BLUR, C[:, 0, 1], C[:, 1, 1] + oaa.BLUR], axis=1)
    J2c = np.zeros((N, 3, 6))
    ab = ((0, 0), (0, 1), (1, 1))
    ij = ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))
    for o, (a, b) in enumerate(ab):
        for e, (i, j) in enumerate(ij):
            v = M[:, a, i] * M[:, b, j]
            if i != j:
                v = v + M[:, a, j] * M[:, b, i]
            J2c[:, o, e] = v
    return c2, J2c, S


def stages(pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy, width, height, model="pinhole", k=None):
    """pose_oracle.stages (+ c2 as aa_oracle.stages, + Jm[N,2,3] the model's du/dpc, 0 on culled rows) for
    any camera model.  A fisheye Gaussian with theta_d' <= 0 is culled like z < 0.2 (depth -1)."""
    if model == "pinhole":
        st = oaa.stages(pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy, width, height)
        st["Jm"] = None
        return st
    _, pcs, depths, _ = orc.project(pws, Rcw, tcw, fx, fy, cx, cy)
    pcs = _f32(pcs).astype(np.float64)
    N = pcs.shape[0]
    keep = depths >= 0.2
    pe = np.where(keep[:, None], pcs, np.array([0.0, 0.0, 1.0]))
    u, J, dJ, valid = project(pe, model, np.float32(fx), np.float32(fy), np.float32(cx), np.float32(cy), k)
    depths = np.where(keep & valid, depths, -1.0)
    d32 = _f32(depths)
    c3, J3r, J3s = orc.compute_cov3d(rots, scales, d32)
    c3 = _f32(c3).astype(np.float64)
    R = _f32(Rcw).astype(np.float64).reshape(3, 3)
    c2, J2c, S = _cov2d(J, R, c3)
    # dcov2d/dpc_c = dJ_c S' J^T + J S' dJ_c^T with S' = R Sigma R^T
    Sp = R[None] @ S @ R.T[None]
    J2p = np.zeros((N, 3, 3))
    for c in range(3):
        D = dJ[:, :, :, c]
        X = D @ Sp @ J.transpose(0, 2, 1)
        X = X + X.transpose(0, 2, 1)
        J2p[:, 0, c], J2p[:, 1, c], J2p[:, 2, c] = X[:, 0, 0], X[:, 0, 1], X[:, 1, 1]
    col, Jcs, Jcp = orc.sh2color(shs, pws, twc)
    cull = d32 < 0.2
    c2[cull] = 0.0
    ci, areas, Jci = orc.inverse_cov2d(_f32(np.where(cull[:, None], 0.0, c2)), d32)
    kept = d32 >= 0.2  # after the NaN-determinant cull
    Ju = np.where(kept[:, None, None], J, 0.0)
    J2c[~kept] = 0.0
    J2p[~kept] = 0.0
    c2[~kept] = 0.0
    us = np.where(kept[:, None], u, 0.0)
    return dict(us=us, ci=ci, col=col, depths=d32, areas=areas, keep=kept, pcs=_f32(pcs), cov3ds=_f32(c3),
                J=(Ju, J3r, J3s, J2c, J2p, Jcs, Jcp, Jci), c2=c2, Jm=Ju)


def camera_grad(st, pws, Rcw, fx, fy, width, height, dloss_dus, dloss_dcinv2ds, dloss_dcolors, dloss_ddepths=None,
                model="pinhole"):
    """pose_oracle.camera_grad of a `stages` result st; with a model other than pinhole the direct term
    J^T dL/dM takes the model's J (st["Jm"])"""
    if model == "pinhole":
        return opose.camera_grad(st, pws, Rcw, fx, fy, width, height, dloss_dus, dloss_dcinv2ds, dloss_dcolors,
                                 dloss_ddepths)
    f = lambda a: np.asarray(a, dtype=np.float64)
    Ju, _, _, _, J2p, _, Jcp, Jci = (f(a) for a in st["J"])
    N = Ju.shape[0]
    R = f(_f32(Rcw)).reshape(3, 3)
    pw = f(_f32(pws)).reshape(N, 3)
    gu, gci, gcol = f(dloss_dus).reshape(N, 2), f(dloss_dcinv2ds).reshape(N, 3), f(dloss_dcolors).reshape(N, 3)
    keep = np.asarray(st["keep"], bool).reshape(N)
    gc2 = np.einsum("ni,nij->nj", gci, Jci)
    gpc = np.einsum("ni,nij->nj", gu, Ju) + np.einsum("ni,nij->nj", gc2, J2p)
    if dloss_ddepths is not None:
        gpc[:, 2] += f(dloss_ddepths).reshape(N)
    gpc[~keep] = 0.0
    c3 = f(st["cov3ds"]).reshape(N, 6)
    J = f(st["Jm"])
    S = c3[:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(N, 3, 3)
    G = np.stack([gc2[:, 0], 0.5 * gc2[:, 1], 0.5 * gc2[:, 1], gc2[:, 2]], axis=1).reshape(N, 2, 2)
    dM = 2.0 * G @ (J @ R[None]) @ S
    dR = np.einsum("nai,naj->nij", J, dM)
    dR[~keep] = 0.0
    per = np.zeros((N, 15))
    per[:, :9] = (gpc[:, :, None] * pw[:, None, :] + dR).reshape(N, 9)
    per[:, 9:12] = gpc
    per[:, 12:15] = -np.einsum("nc,ncb->nb", gcol, Jcp)
    return dict(grad=per.sum(0), per=per, absum=np.abs(per).sum(0))


def step(scene, cam, *, rgbd, pose, aa, filt, dl, dld=None, dla=None, drawn_inputs=None, model="pinhole", k=None):
    """step_oracle.step for any camera model (pinhole: step_oracle.step itself).  The flagged rows are
    step_oracle's (rasterizer-ambiguous, near-plane band, thin, AA) plus, for the fisheye, the rows within
    1e-4 (relative) of the theta_d' <= 0 cull."""
    if model == "pinhole":
        return ostep.step(scene, cam, rgbd=rgbd, pose=pose, aa=aa, filt=filt, dl=dl, dld=dld, dla=dla,
                          drawn_inputs=drawn_inputs)
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
    if model == "fisheye":
        P1 = fisheye_terms(pc64, k)["P1"]
        band |= np.abs(P1) < 1e-4
    thin = oaa.thin(sf)
    flagged = amb | band | thin
    if aa:
        flagged = flagged | oaa.flagged(sf, s)
    return dict(image=out["image"], depth=out.get("depth"), alpha=out.get("alpha"), ambiguous=out["ambiguous"],
                grads=g, raster=(du, dc, da, dcol, dz), per=per, absum=np.abs(per).sum(0), cam_grad=per.sum(0),
                flagged=flagged, thin=thin, band=band, st=st, rho=rho, drawn=rho * af)
