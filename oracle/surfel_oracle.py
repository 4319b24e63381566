"""fp64 numpy oracle of 2D Gaussian Splatting (DESIGN 3.15).  TEST INFRASTRUCTURE ONLY.

The model of the surfel kernels, stated once more in double precision: per-surfel stages
(`preprocess`), a tile-exact compositor (`render`: oracle.bin's tiles and depth order, the clamp,
skip and stop rules of the colour path), its analytic backward into the kernels' gradient rows
(`render_backward`) and the rows into parameter gradients (`preprocess_backward`).  `delta`
shifts every surfel in screen space (evaluated at p - delta): its gradient at 0 is the rows'
dL/ddelta.  Pixels whose result hangs on a threshold within `margin` are flagged ambiguous.
"""
import numpy as np

from . import oracle as orc

ALPHA_CLAMP, ALPHA_SKIP, TAU_STOP = 0.99, 0.002, 1e-4
FILTER = 2.0    # G2 = 2 |p - u|^2
CUTOFF2 = 9.0   # the binning footprint: a^2 + b^2 <= 9
AREA_CAP = 2 ** 24  # binning half-extents at or above it are clamped to it, not culled

_C1 = 0.4886025119029199
_C20, _C22, _C24 = 1.0925484305920792, 0.31539156525252005, 0.5462742152960396
_C30, _C31, _C32, _C33, _C35 = -0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, \
    1.445305721320277


def sh_basis(r, k):
    """Y[N,k] and dY[N,k,3] (partials of the polynomials in x, y, z), pg::sh_basis in fp64"""
    x, y, z = r[:, 0], r[:, 1], r[:, 2]
    o, l = np.zeros_like(x), np.ones_like(x)
    xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
    rows = [(0.28209479177387814 * l, o, o, o), (-_C1 * y, o, -_C1 * l, o), (_C1 * z, o, o, _C1 * l),
            (-_C1 * x, -_C1 * l, o, o),
            (_C20 * xy, _C20 * y, _C20 * x, o), (-_C20 * yz, o, -_C20 * z, -_C20 * y),
            (_C22 * (2 * zz - xx - yy), -2 * _C22 * x, -2 * _C22 * y, 4 * _C22 * z), (-_C20 * xz, -_C20 * z, o, -_C20 * x),
            (_C24 * (xx - yy), 2 * _C24 * x, -2 * _C24 * y, o),
            (_C30 * y * (3 * xx - yy), _C30 * 6 * xy, _C30 * (3 * xx - 3 * yy), o), (_C31 * xy * z, _C31 * yz, _C31 * xz, _C31 * xy),
            (_C32 * y * (4 * zz - xx - yy), _C32 * (-2 * xy), _C32 * (4 * zz - xx - 3 * yy), _C32 * 8 * yz),
            (_C33 * z * (2 * zz - 3 * xx - 3 * yy), _C33 * (-6 * xz), _C33 * (-6 * yz), _C33 * (6 * zz - 3 * xx - 3 * yy)),
            (_C32 * x * (4 * zz - xx - yy), _C32 * (4 * zz - 3 * xx - yy), _C32 * (-2 * xy), _C32 * 8 * xz),
            (_C35 * z * (xx - yy), _C35 * 2 * xz, _C35 * (-2 * yz), _C35 * (xx - yy)),
            (_C30 * x * (xx - 3 * yy), _C30 * (3 * xx - 3 * yy), _C30 * (-6 * xy), o)][:k]
    Y = np.stack([r_[0] for r_ in rows], 1)
    dY = np.stack([np.stack(r_[1:], 1) for r_ in rows], 1)
    return Y, dY


def quat_R(q):
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                     2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                     2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)


def footprint(M, u, lv):
    """half-extents around u of the boxes of {a^2 + b^2 <= lv} through M and {2|p-u|^2 <= lv};
    -> (ext[N,2], bounded[N])"""
    D = M[:, 2, 2] ** 2 - lv * (M[:, 2, 0] ** 2 + M[:, 2, 1] ** 2)
    ok = D > 0
    Di = np.where(ok, 1.0 / np.where(ok, D, 1.0), 0.0)
    ext = np.zeros((M.shape[0], 2))
    r = np.sqrt(lv / FILTER)
    for k in range(2):
        m = M[:, k]
        cen = (m[:, 2] * M[:, 2, 2] - lv * (m[:, 0] * M[:, 2, 0] + m[:, 1] * M[:, 2, 1])) * Di
        hh = cen * cen - (m[:, 2] ** 2 - lv * (m[:, 0] ** 2 + m[:, 1] ** 2)) * Di
        h = np.sqrt(np.maximum(hh, 0))
        ext[:, k] = np.maximum(np.maximum(np.abs(cen + h - u[:, k]), np.abs(cen - h - u[:, k])), r)
    return ext, ok


def preprocess(pws, rots, scales, shs, Rcw, tcw, twc, fx, fy, cx, cy):
    """per-surfel stages -> dict(M[N,3,3], u[N,2], depths[N] (-1 culled), areas[N,2] i32 (at most AREA_CAP),
    ext[N,2] (the fp64 binning half-extents),
    colors[N,3], n[N,3], keep[N], and what the backward needs)"""
    f = lambda a: np.asarray(a, dtype=np.float64)
    pws, rots, scales, shs = f(pws), f(rots), f(scales), f(shs).reshape(len(pws), -1)
    Rcw, tcw, twc = f(Rcw).reshape(3, 3), f(tcw).reshape(3), f(twc).reshape(3)
    N, k = len(pws), shs.shape[1] // 3
    pc = pws @ Rcw.T + tcw
    qnorm = np.linalg.norm(rots, axis=1)
    qn = rots / qnorm[:, None]
    R = quat_R(qn)
    axes = np.einsum("ij,njk->nik", Rcw, R)  # camera-frame R e_k in column k
    tu, tv = scales[:, :1] * axes[:, :, 0], scales[:, 1:2] * axes[:, :, 1]
    sgn = np.where(np.sum(axes[:, :, 2] * pc, 1) > 0, -1.0, 1.0)
    n = sgn[:, None] * axes[:, :, 2]
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])
    M = np.einsum("ij,njk->nik", K, np.stack([tu, tv, pc], 2))
    keep = pc[:, 2] >= np.float32(0.2)
    z = np.where(keep, pc[:, 2], 1.0)
    u = np.stack([fx * pc[:, 0] / z + cx, fy * pc[:, 1] / z + cy], 1)
    ext, ok = footprint(M, u, CUTOFF2)
    keep &= ok
    areas = np.where(keep[:, None], np.where(ext < AREA_CAP, np.ceil(np.minimum(ext, AREA_CAP)), AREA_CAP), 0)
    areas = areas.astype(np.int32)
    d = pws - twc
    dn = np.linalg.norm(d, axis=1)
    r = d / dn[:, None] if k > 1 else np.zeros_like(d)
    Y, dY = sh_basis(r, k)
    col = 0.5 + np.einsum("nl,nlc->nc", Y, shs.reshape(N, k, 3))
    return dict(M=M, u=np.where(keep[:, None], u, 0), depths=np.where(keep, pc[:, 2], -1.0), areas=areas, ext=ext,
                colors=col, n=n, keep=keep, pc=pc, qn=qn, qnorm=qnorm, R=R, axes=axes, sgn=sgn, scales=scales,
                Y=Y, dY=dY, r=r, dn=dn, shs=shs, Rcw=Rcw, K=K, k=k)


def _eval(M, u, X, Y):
    """one surfel at pixels (X, Y): the plane point, which term wins and the hit depth"""
    hx = X[:, None] * M[2] - M[0]
    hy = Y[:, None] * M[2] - M[1]
    c = np.cross(hx, hy)
    with np.errstate(divide="ignore", invalid="ignore"):
        a, b = c[:, 0] / c[:, 2], c[:, 1] / c[:, 2]
        G3 = np.where(c[:, 2] != 0, a * a + b * b, np.inf)
    G3 = np.where(np.isnan(G3), np.inf, G3)
    dx, dy = X - u[0], Y - u[1]
    G2 = FILTER * (dx * dx + dy * dy)
    b3 = G3 <= G2
    G = np.where(b3, G3, G2)
    z = np.where(b3, M[2, 0] * np.where(b3, a, 0) + M[2, 1] * np.where(b3, b, 0) + M[2, 2], M[2, 2])
    return dict(hx=hx, hy=hy, c=c, a=a, b=b, b3=b3, G=G, G3=G3, G2=G2, z=z, dx=dx, dy=dy)


def _tiles(H, W, ranges):
    gx = (W + 15) // 16
    for t in range(len(ranges)):
        if ranges[t, 1] <= ranges[t, 0]:
            continue
        x0, y0 = (t % gx) * 16, (t // gx) * 16
        ys, xs = np.mgrid[y0:min(y0 + 16, H), x0:min(x0 + 16, W)]
        yield t, xs.ravel(), ys.ravel()


def render(H, W, pre, alphas, bins, delta=None, margin=2e-5):
    """front-to-back compositing of the binned surfels; bins = oracle.bin(...)'s (P, ranges, gsid, keys).
    -> dict(image[3,H,W], depth, alpha, normal[3,H,W], contrib, final_tau, ambiguous[H,W])"""
    alphas = np.asarray(alphas, dtype=np.float64).reshape(-1)
    _, ranges, gsid, _ = bins
    out = dict(image=np.zeros((3, H, W)), depth=np.zeros((H, W)), alpha=np.zeros((H, W)),
               normal=np.zeros((3, H, W)), contrib=np.zeros((H, W), np.int32), final_tau=np.zeros((H, W)),
               ambiguous=np.zeros((H, W), bool))
    for t, X, Y in _tiles(H, W, ranges):
        Xf, Yf = X.astype(np.float64), Y.astype(np.float64)
        tau = np.ones(len(X))
        acc = np.zeros((8, len(X)))
        cont = np.zeros(len(X), np.int32)
        amb = np.zeros(len(X), bool)
        for j, i in enumerate(gsid[ranges[t, 0]:ranges[t, 1]]):
            sh = (0.0, 0.0) if delta is None else delta[i]
            e = _eval(pre["M"][i], pre["u"][i], Xf - sh[0], Yf - sh[1])
            ag = alphas[i] * np.exp(-0.5 * e["G"])
            ap = np.minimum(ALPHA_CLAMP, ag)
            on = (tau >= TAU_STOP) & (ap >= ALPHA_SKIP)
            live = tau >= TAU_STOP * (1 - margin)
            amb |= live & ((np.abs(ap - ALPHA_SKIP) < margin * ALPHA_SKIP) | (np.abs(ag - ALPHA_CLAMP) < margin) |
                           (np.abs(e["G3"] - e["G2"]) < margin * np.maximum(1.0, e["G2"])))
            amb |= (ap >= ALPHA_SKIP) & (np.abs(tau - TAU_STOP) < margin * TAU_STOP)
            w = np.where(on, tau * ap, 0.0)
            vals = np.concatenate([pre["colors"][i][:, None] * np.ones(len(X)), e["z"][None], np.ones((1, len(X))),
                                   pre["n"][i][:, None] * np.ones(len(X))])
            acc += w * vals
            tau = np.where(on, tau * (1 - ap), tau)
            cont = np.where(on, j + 1, cont)
        out["image"][:, Y, X] = acc[:3]
        out["depth"][Y, X] = acc[3]
        out["alpha"][Y, X] = acc[4]
        out["normal"][:, Y, X] = acc[5:]
        out["contrib"][Y, X] = cont
        out["final_tau"][Y, X] = tau
        out["ambiguous"][Y, X] = amb
    return out


def render_backward(H, W, pre, alphas, bins, fwd, dl_image, dl_depth, dl_alpha, dl_normal, abs_rows=False):
    """the analytic backward of `render` on its own forward state -> rows[N,18] =
    [dL/dM (row-major 9), dL/dalpha, dL/dcolour (3), dL/dn (3), dL/ddelta (2)], dL/du folded into dL/dM.
    abs_rows: also -> the same rows summed over the absolute values of every per-pixel product that
    makes up an entry (the scale of an fp32 sum's rounding: the conditioning of that entry)"""
    alphas = np.asarray(alphas, dtype=np.float64).reshape(-1)
    N = len(alphas)
    _, ranges, gsid, _ = bins
    z2 = lambda a, s: np.zeros(s) if a is None else np.asarray(a, dtype=np.float64).reshape(s)
    dli, dld, dla, dln = z2(dl_image, (3, H, W)), z2(dl_depth, (H, W)), z2(dl_alpha, (H, W)), z2(dl_normal, (3, H, W))
    rows = np.zeros((N, 18))
    absr = np.zeros((N, 18))
    across = lambda p, q: np.stack([p[:, 1] * q[:, 2] + p[:, 2] * q[:, 1], p[:, 2] * q[:, 0] + p[:, 0] * q[:, 2],
                                    p[:, 0] * q[:, 1] + p[:, 1] * q[:, 0]], 1)
    for t, X, Y in _tiles(H, W, ranges):
        Xf, Yf = X.astype(np.float64), Y.astype(np.float64)
        tau = fwd["final_tau"][Y, X].copy()
        cont = fwd["contrib"][Y, X]
        D = np.concatenate([dli[:, Y, X], dld[None, Y, X], dla[None, Y, X], dln[:, Y, X]])
        sdot, sabs = np.zeros(len(X)), np.zeros(len(X))
        ids = gsid[ranges[t, 0]:ranges[t, 1]]
        for j in range(len(ids) - 1, -1, -1):
            i = ids[j]
            M, u = pre["M"][i], pre["u"][i]
            e = _eval(M, u, Xf, Yf)
            g = np.exp(-0.5 * e["G"])
            ag = alphas[i] * g
            ap = np.minimum(ALPHA_CLAMP, ag)
            on = (j < cont) & (ap >= ALPHA_SKIP)
            if not on.any():
                continue
            ap = np.where(on, ap, 0.0)
            tau = tau / (1 - ap)
            vals = np.concatenate([pre["colors"][i][:, None] * np.ones(len(X)), e["z"][None], np.ones((1, len(X))),
                                   pre["n"][i][:, None] * np.ones(len(X))])
            v = np.sum(D * vals, 0)
            diff = v - sdot
            sdot = sdot + ap * diff
            dap = np.where(on, tau * diff, 0.0)
            vabs = np.sum(np.abs(D * vals), 0)
            dapm = np.where(on, tau * (vabs + sabs), 0.0)  # |dL/dalpha'| before its cancellations
            sabs = sabs + ap * (vabs + sabs)
            w = tau * ap
            unc = on & (ag <= ALPHA_CLAMP)
            dG = np.where(unc, -0.5 * dap * ap, 0.0)
            dz = w * D[3]
            b3 = e["b3"] & on
            a, b = np.where(b3, e["a"], 0), np.where(b3, e["b"], 0)
            da = np.where(b3, dG * 2 * a + dz * M[2, 0], 0)
            db = np.where(b3, dG * 2 * b + dz * M[2, 1], 0)
            c2 = np.where(b3, e["c"][:, 2], 1.0)
            gc = np.stack([da / c2, db / c2, -(da * a + db * b) / c2], 1)
            ex = np.cross(e["hy"], gc)
            ey = np.cross(gc, e["hx"])
            kk = np.where(on & ~e["b3"], -2 * FILTER * dG, 0)
            # u = (m1z, m2z) / m3z: the filter branch's dL/du folded into dL/dM
            zi = 1.0 / M[2, 2]
            gux, guy = kk * e["dx"], kk * e["dy"]
            # every entry as a sum of per-pixel terms; mag: the size of the products inside a term
            # (ex, ey are cross products of h with dL/dc, and dL/dc is made of dL/da, dL/db)
            dGm = np.where(unc, 0.5 * dapm * ap, 0.0)
            dam = np.where(b3, dGm * 2 * np.abs(a) + np.abs(dz * M[2, 0]), 0)
            dbm = np.where(b3, dGm * 2 * np.abs(b) + np.abs(dz * M[2, 1]), 0)
            aga = np.stack([dam, dbm, dam * np.abs(a) + dbm * np.abs(b)], 1) / np.abs(c2)[:, None]
            guxm, guym = np.where(kk != 0, 2 * FILTER * dGm, 0) * np.abs(e["dx"]), \
                np.where(kk != 0, 2 * FILTER * dGm, 0) * np.abs(e["dy"])
            exa, eya = across(np.abs(e["hy"]), aga), across(aga, np.abs(e["hx"]))

            def add(k, term, mag=None):
                rows[i, k] += np.sum(term)
                absr[i, k] += np.sum(np.abs(term) if mag is None else mag)

            for k in range(3):
                add(k, -ex[:, k], exa[:, k])
                add(3 + k, -ey[:, k], eya[:, k])
                add(6 + k, Xf * ex[:, k], Xf * exa[:, k])
                add(6 + k, Yf * ey[:, k], Yf * eya[:, k])
                add(16, -ex[:, k] * M[2, k], exa[:, k] * abs(M[2, k]))
                add(17, -ey[:, k] * M[2, k], eya[:, k] * abs(M[2, k]))
                add(10 + k, w * D[k])
                add(13 + k, w * D[5 + k])
            add(6, dz * a)
            add(7, dz * b)
            add(8, dz)
            add(2, gux * zi, guxm * abs(zi))
            add(5, guy * zi, guym * abs(zi))
            add(8, -(gux * M[0, 2] + guy * M[1, 2]) * zi * zi, (guxm * abs(M[0, 2]) + guym * abs(M[1, 2])) * zi * zi)
            add(9, np.where(unc, dap * g, 0), np.where(unc, dapm * g, 0))
            add(16, gux, guxm)
            add(17, guy, guym)
    return (rows, absr) if abs_rows else rows


def preprocess_backward(pre, rows, twc=None):
    """rows[N,18] -> dict(pws, shs, alphas, scales, rots, us) in fp64"""
    N, k = len(rows), pre["k"]
    gcol = rows[:, 10:13]
    Y, dY, r, dn = pre["Y"], pre["dY"], pre["r"], pre["dn"]
    shs = pre["shs"].reshape(N, k, 3)
    dshs = (Y[:, :, None] * gcol[:, None, :]).reshape(N, -1)
    gpw = np.zeros((N, 3))
    if k > 1:
        t = np.einsum("nlc,nc->nl", shs, gcol)
        gdir = np.einsum("nl,nld->nd", t[:, 1:], dY[:, 1:])
        rg = np.sum(r * gdir, 1)
        gpw = (gdir - r * rg[:, None]) / dn[:, None]
    K, Rcw = pre["K"], pre["Rcw"]
    gMs = rows[:, :9].reshape(N, 3, 3)
    gX = np.einsum("ji,njk->nik", K, gMs)  # K^T dL/dM: columns tu, tv, pc
    keep = pre["keep"]
    gpw += np.where(keep[:, None], gX[:, :, 2] @ Rcw, 0)
    s = pre["scales"]
    gcam = [gX[:, :, 0], gX[:, :, 1], rows[:, 13:16]]
    sc = [s[:, 0], s[:, 1], pre["sgn"]]
    gw = [sc[j][:, None] * (gcam[j] @ Rcw) for j in range(3)]  # world-frame dL/d(R e_j)
    R = pre["R"]
    gs = np.zeros((N, 3))
    for j in range(2):
        gs[:, j] = np.sum((gX[:, :, j] @ Rcw) * R[:, :, j], 1)
    dR = np.stack(gw, 2)  # dR[n, a, j] = dL/dR_aj
    w, x, y, z = pre["qn"].T
    d = dR.reshape(N, 9).T
    gn = np.stack([2 * (-z * d[1] + y * d[2] + z * d[3] - x * d[5] - y * d[6] + x * d[7]),
                   2 * (y * d[1] + z * d[2] + y * d[3] - 2 * x * d[4] - w * d[5] + z * d[6] + w * d[7] - 2 * x * d[8]),
                   2 * (-2 * y * d[0] + x * d[1] + w * d[2] + x * d[3] + z * d[5] - w * d[6] + z * d[7] - 2 * y * d[8]),
                   2 * (-2 * z * d[0] - w * d[1] + x * d[2] + w * d[3] - 2 * z * d[4] + y * d[5] + x * d[6] + y * d[7])], 1)
    qn = pre["qn"]
    grots = (gn - qn * np.sum(qn * gn, 1)[:, None]) / pre["qnorm"][:, None]
    kp = keep[:, None]
    return dict(pws=gpw, shs=dshs, alphas=rows[:, 9], scales=np.where(kp, gs, 0), rots=np.where(kp, grots, 0),
                us=rows[:, 16:18])


def bin_f32(H, W, pre):
    """oracle.bin on the fp32 (u, depths, areas) of `pre` (copies: bin mutates its inputs)"""
    return orc.bin(H, W, pre["u"].astype(np.float32), pre["depths"].astype(np.float32).copy(),
                   np.ascontiguousarray(pre["areas"], dtype=np.int32).copy())
