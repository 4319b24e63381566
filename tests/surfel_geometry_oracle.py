"""fp64 model of the 2DGS geometry terms (DESIGN 3.16).  TEST INFRASTRUCTURE ONLY.

oracle/surfel_oracle.py's compositor with the depth-distortion and median-depth planes of
k_draw_2dgs (`render_geometry`) and its analytic backward with their gradients, as
k_draw_2dgs_bwd adds them (`render_backward_geometry`).  The surfel planes, the binning, the
rows' layout and `preprocess` / `preprocess_backward` are surfel_oracle's.

Per pixel, over the contributing records in compositing order (w = tau alpha', z the hit depth):
    m(z) = far / (far - near) (1 - near / max(z, near))
    distortion = sum_{j<i} w_i w_j (m_i - m_j)^2, accumulated as w_i (m_i^2 A + D2 - 2 m_i D) before
                 record i joins A = sum w, D = sum w m, D2 = sum w m^2
    median = z of the last record whose incoming tau > 0.5 (median_contrib: its index + 1)
"""
import numpy as np

from oracle import surfel_oracle as so


def m_of(z, near, far):
    return far / (far - near) * (1.0 - near / np.maximum(z, near))


def dm_of(z, near, far):
    return np.where(z > near, far / (far - near) * near / np.where(z > near, z, 1.0) ** 2, 0.0)


def render_geometry(H, W, pre, alphas, bins, near=0.2, far=100.0, delta=None, margin=2e-5, exact=False):
    """so.render's planes plus distortion[H,W], moments[2,H,W] = (D, D2), median_depth[H,W],
    median_contrib[H,W] i32 and count[H,W] i32 (the contributing records).  `ambiguous` also flags
    pixels where a contributing record's incoming tau lies within margin of 0.5 or its hit depth within
    margin of near.  exact: a tau of exactly 0.5 or a hit depth of exactly near is not flagged (scenes
    built so that fp32 computes the same values); the pixels where one occurs are returned as
    ties[H,W] and at_near[H,W]."""
    out = so.render(H, W, pre, alphas, bins, delta=delta, margin=margin)
    alphas = np.asarray(alphas, dtype=np.float64).reshape(-1)
    _, ranges, gsid, _ = bins
    out.update(distortion=np.zeros((H, W)), moments=np.zeros((2, H, W)), median_depth=np.zeros((H, W)),
               median_contrib=np.zeros((H, W), np.int32), count=np.zeros((H, W), np.int32),
               ties=np.zeros((H, W), bool), at_near=np.zeros((H, W), bool))
    for t, X, Y in so._tiles(H, W, ranges):
        Xf, Yf = X.astype(np.float64), Y.astype(np.float64)
        tau = np.ones(len(X))
        A, D, D2, dist, medz = (np.zeros(len(X)) for _ in range(5))
        medc, cnt = np.zeros(len(X), np.int32), np.zeros(len(X), np.int32)
        amb, tie, atn = np.zeros(len(X), bool), np.zeros(len(X), bool), np.zeros(len(X), bool)
        for j, i in enumerate(gsid[ranges[t, 0]:ranges[t, 1]]):
            sh = (0.0, 0.0) if delta is None else delta[i]
            e = so._eval(pre["M"][i], pre["u"][i], Xf - sh[0], Yf - sh[1])
            ap = np.minimum(so.ALPHA_CLAMP, alphas[i] * np.exp(-0.5 * e["G"]))
            on = (tau >= so.TAU_STOP) & (ap >= so.ALPHA_SKIP)
            t5, zn = on & (tau == 0.5), on & (e["z"] == near)
            amb |= on & (((np.abs(tau - 0.5) < margin) & ~(exact & t5)) |
                         ((np.abs(e["z"] - near) < margin * max(1.0, near)) & ~(exact & zn)))
            tie |= t5
            atn |= zn
            cnt += on
            w = np.where(on, tau * ap, 0.0)
            m = np.where(on, m_of(e["z"], near, far), 0.0)
            dist += w * (m * m * A + D2 - 2 * m * D)
            A += w
            D += w * m
            D2 += w * m * m
            med = on & (tau > 0.5)
            medz = np.where(med, e["z"], medz)
            medc = np.where(med, j + 1, medc)
            tau = np.where(on, tau * (1 - ap), tau)
        out["distortion"][Y, X] = dist
        out["moments"][:, Y, X] = np.stack([D, D2])
        out["median_depth"][Y, X] = medz
        out["median_contrib"][Y, X] = medc
        out["count"][Y, X] = cnt
        out["ambiguous"][Y, X] |= amb
        out["ties"][Y, X] = tie
        out["at_near"][Y, X] = atn
    return out


def render_backward_geometry(H, W, pre, alphas, bins, fwd, dl_image=None, dl_depth=None, dl_alpha=None,
                             dl_normal=None, dl_distortion=None, dl_median=None, near=0.2, far=100.0,
                             abs_rows=False):
    """so.render_backward with the geometry terms: per contributing (record i, pixel), the per-record
    value of the alpha' recurrence gains dL/ddistortion (m_i^2 A + D2 - 2 m_i D) and the hit-depth
    coefficient gains dL/ddistortion 2 w_i (m_i A - D) m'(z_i) + dL/dmedian [i is the median record]
    (A, D, D2 the pixel's final totals).  -> rows[N,18] (and abs_rows, the conditioning, as there)"""
    alphas = np.asarray(alphas, dtype=np.float64).reshape(-1)
    N = len(alphas)
    _, ranges, gsid, _ = bins
    z2 = lambda a, s: np.zeros(s) if a is None else np.asarray(a, dtype=np.float64).reshape(s)
    dli, dld, dla, dln = z2(dl_image, (3, H, W)), z2(dl_depth, (H, W)), z2(dl_alpha, (H, W)), z2(dl_normal, (3, H, W))
    dlx, dlm = z2(dl_distortion, (H, W)), z2(dl_median, (H, W))
    rows = np.zeros((N, 18))
    absr = np.zeros((N, 18))
    across = lambda p, q: np.stack([p[:, 1] * q[:, 2] + p[:, 2] * q[:, 1], p[:, 2] * q[:, 0] + p[:, 0] * q[:, 2],
                                    p[:, 0] * q[:, 1] + p[:, 1] * q[:, 0]], 1)
    for t, X, Y in so._tiles(H, W, ranges):
        Xf, Yf = X.astype(np.float64), Y.astype(np.float64)
        tau = fwd["final_tau"][Y, X].copy()
        cont = fwd["contrib"][Y, X]
        A, D, D2 = fwd["alpha"][Y, X], fwd["moments"][0, Y, X], fwd["moments"][1, Y, X]
        medc = fwd["median_contrib"][Y, X]
        gx_, gm_ = dlx[Y, X], dlm[Y, X]
        Dp = np.concatenate([dli[:, Y, X], dld[None, Y, X], dla[None, Y, X], dln[:, Y, X]])
        sdot, sabs = np.zeros(len(X)), np.zeros(len(X))
        ids = gsid[ranges[t, 0]:ranges[t, 1]]
        for j in range(len(ids) - 1, -1, -1):
            i = ids[j]
            M, u = pre["M"][i], pre["u"][i]
            e = so._eval(M, u, Xf, Yf)
            g = np.exp(-0.5 * e["G"])
            ag = alphas[i] * g
            ap = np.minimum(so.ALPHA_CLAMP, ag)
            on = (j < cont) & (ap >= so.ALPHA_SKIP)
            if not on.any():
                continue
            ap = np.where(on, ap, 0.0)
            tau = tau / (1 - ap)
            vals = np.concatenate([pre["colors"][i][:, None] * np.ones(len(X)), e["z"][None], np.ones((1, len(X))),
                                   pre["n"][i][:, None] * np.ones(len(X))])
            m = m_of(e["z"], near, far)
            vg = gx_ * (m * m * A + D2 - 2 * m * D)
            v = np.sum(Dp * vals, 0) + vg
            diff = v - sdot
            sdot = sdot + ap * diff
            dap = np.where(on, tau * diff, 0.0)
            vabs = np.sum(np.abs(Dp * vals), 0) + np.abs(gx_) * (m * m * A + D2 + 2 * m * D)
            dapm = np.where(on, tau * (vabs + sabs), 0.0)
            sabs = sabs + ap * (vabs + sabs)
            w = tau * ap
            unc = on & (ag <= so.ALPHA_CLAMP)
            dG = np.where(unc, -0.5 * dap * ap, 0.0)
            dm = dm_of(e["z"], near, far)
            dz = w * Dp[3] + gx_ * 2 * w * (m * A - D) * dm + np.where(medc == j + 1, gm_, 0.0)
            dzm = np.abs(w * Dp[3]) + np.abs(gx_) * 2 * w * (m * A + D) * dm + np.where(medc == j + 1, np.abs(gm_), 0)
            dz, dzm = np.where(on, dz, 0.0), np.where(on, dzm, 0.0)
            b3 = e["b3"] & on
            a, b = np.where(b3, e["a"], 0), np.where(b3, e["b"], 0)
            da = np.where(b3, dG * 2 * a + dz * M[2, 0], 0)
            db = np.where(b3, dG * 2 * b + dz * M[2, 1], 0)
            c2 = np.where(b3, e["c"][:, 2], 1.0)
            gc = np.stack([da / c2, db / c2, -(da * a + db * b) / c2], 1)
            ex = np.cross(e["hy"], gc)
            ey = np.cross(gc, e["hx"])
            kk = np.where(on & ~e["b3"], -2 * so.FILTER * dG, 0)
            zi = 1.0 / M[2, 2]
            gux, guy = kk * e["dx"], kk * e["dy"]
            dGm = np.where(unc, 0.5 * dapm * ap, 0.0)
            dam = np.where(b3, dGm * 2 * np.abs(a) + dzm * abs(M[2, 0]), 0)
            dbm = np.where(b3, dGm * 2 * np.abs(b) + dzm * abs(M[2, 1]), 0)
            aga = np.stack([dam, dbm, dam * np.abs(a) + dbm * np.abs(b)], 1) / np.abs(c2)[:, None]
            guxm, guym = np.where(kk != 0, 2 * so.FILTER * dGm, 0) * np.abs(e["dx"]), \
                np.where(kk != 0, 2 * so.FILTER * dGm, 0) * np.abs(e["dy"])
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
                add(10 + k, w * Dp[k])
                add(13 + k, w * Dp[5 + k])
            add(6, dz * a, dzm * np.abs(a))
            add(7, dz * b, dzm * np.abs(b))
            add(8, dz, dzm)
            add(2, gux * zi, guxm * abs(zi))
            add(5, guy * zi, guym * abs(zi))
            add(8, -(gux * M[0, 2] + guy * M[1, 2]) * zi * zi, (guxm * abs(M[0, 2]) + guym * abs(M[1, 2])) * zi * zi)
            add(9, np.where(unc, dap * g, 0), np.where(unc, dapm * g, 0))
            add(16, gux, guxm)
            add(17, guy, guym)
    return (rows, absr) if abs_rows else rows


def composited_at(H, W, pre, alphas, bins, fwd, mask):
    """bool[N]: the surfels with a contributing record (list position < contrib, alpha' >= the skip
    threshold) at some pixel of mask[H,W]"""
    alphas = np.asarray(alphas, dtype=np.float64).reshape(-1)
    _, ranges, gsid, _ = bins
    hit = np.zeros(len(alphas), bool)
    for t, X, Y in so._tiles(H, W, ranges):
        m = mask[Y, X]
        if not m.any():
            continue
        X, Y = X[m], Y[m]
        cont = fwd["contrib"][Y, X]
        for j, i in enumerate(gsid[ranges[t, 0]:ranges[t, 1]]):
            if hit[i] or j >= cont.max():
                continue
            e = so._eval(pre["M"][i], pre["u"][i], X.astype(np.float64), Y.astype(np.float64))
            ap = np.minimum(so.ALPHA_CLAMP, alphas[i] * np.exp(-0.5 * e["G"]))
            hit[i] = ((j < cont) & (ap >= so.ALPHA_SKIP)).any()
    return hit


def brute_force(ws, ms, zs, taus_in, idxs):
    """one pixel's distortion (the O(K^2) double sum) and median (scanning the incoming taus) from its
    contributing records' weights, mapped depths, hit depths, incoming taus and patch indices"""
    K = len(ws)
    dist = sum(ws[i] * ws[j] * (ms[i] - ms[j]) ** 2 for i in range(K) for j in range(i))
    med, medc = 0.0, 0
    for i in range(K):
        if taus_in[i] > 0.5:
            med, medc = zs[i], idxs[i] + 1
    return dist, med, medc
