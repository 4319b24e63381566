"""fp64 oracle of feature rendering: per-Gaussian features f_i in R^D composited with the image's
weights, F[c, p] = sum_i w_i(p) f_i[c].  TEST INFRASTRUCTURE ONLY.

No derivative code of its own.  F is the colour oracle's image with the colours replaced by a triple
of feature channels; the forward state (contrib, final_tau, ranges, gsid) does not depend on the
colours, and the rasterizer backward is linear in its upstream gradient for a fixed forward state.
So the feature oracle is `oracle.splat` / `oracle.splat_backward` run once per channel triple (the
last one zero-padded) and summed; the dcol of triple k is dL/dfeatures[:, 3k:3k+3].
`step_features` is `step_oracle.step` (colour, no pose, no RGB-D) with the feature terms added to
the rasterizer gradients before the shared chain.
"""
import numpy as np

from . import aa_oracle as oaa
from . import filter3d_oracle as of3
from . import oracle as orc
from . import step_oracle as ost


def _triples(a, D):
    """[..., D] -> list of [..., 3] column triples, the last zero-padded"""
    a = np.asarray(a, np.float64)
    pad = (-D) % 3
    if pad:
        a = np.concatenate([a, np.zeros(a.shape[:-1] + (pad,))], axis=-1)
    return [a[..., 3 * k:3 * k + 3] for k in range((D + pad) // 3)]


def splat_features(height, width, us, cinv2ds, alphas, depths, areas, features, margin=2e-5):
    """`oracle.splat` with features[N, D] in place of the colours.  depths / areas are copied (the
    binning culls in place).  -> dict(features[D,H,W] f64, contrib, final_tau, ranges, gsid, keys, P,
    ambiguous[H,W] (the union over the triples -- identical, they share the forward state))"""
    f = np.asarray(features, np.float32)
    N, D = f.shape
    out, planes = None, []
    for trip in _triples(f.astype(np.float64), D):
        o = orc.splat(height, width, us, cinv2ds, alphas, np.array(depths, np.float32).reshape(-1),
                      np.ascontiguousarray(trip, np.float32), np.array(areas, np.int32), margin=margin)
        planes.append(o["image"])
        if out is None:
            out = o
        else:
            out["ambiguous"] = out["ambiguous"] | o["ambiguous"]
    res = dict(out)
    res.pop("image")
    res["features"] = np.concatenate(planes, axis=0)[:D]
    return res


def splat_backward_features(height, width, us, cinv2ds, alphas, fwd, features, dloss_dfeatures_map,
                            return_ambiguous=False, margin=2e-5, rows=False):
    """Backward of `splat_features` on the forward state `fwd` (contrib, final_tau, ranges, gsid):
    dL/dF [D,H,W] -> dloss_dus[N,1,2], dloss_dcinv2ds[N,1,3], dloss_dalphas[N,1,1] (the sums over
    the triples) and dloss_dfeatures[N,D] (+ bool[N], the union of the triples' ambiguity flags).
    rows: instead, the moment rows k_draw_feat_bwd adds (`oracle.splat_backward_rows`' dict summed over
    the triples; rows 6-8 zero) and dfeatures[N,D] with dfeatures_abs / _maha / _amb.  Every conditioning
    sum is linear in the per-channel magnitudes, so the triples' sums are the all-channel ones."""
    f = np.asarray(features, np.float32)
    N, D = f.shape
    dl = np.asarray(dloss_dfeatures_map, np.float64)
    dl_t = _triples(np.moveaxis(dl, 0, -1), D)  # [H,W,3] each
    if rows:
        out = None
        dfeat = [np.zeros((N, len(dl_t) * 3)) for _ in range(4)]
        for k, (trip, g) in enumerate(zip(_triples(f.astype(np.float64), D), dl_t)):
            r = orc.splat_backward_rows(height, width, us, cinv2ds, alphas, np.ascontiguousarray(trip, np.float32),
                                        fwd, np.ascontiguousarray(np.moveaxis(g, -1, 0), np.float32), margin=margin)
            for j, key in enumerate(("rows", "abs_rows", "maha_rows", "amb_rows")):
                dfeat[j][:, 3 * k:3 * k + 3] = r[key][:, 6:9]
                r[key][:, 6:9] = 0
            if out is None:
                out = r
            else:
                for key in ("rows", "abs_rows", "maha_rows", "amb_rows"):
                    out[key] = out[key] + r[key]
                out["ambiguous"] = out["ambiguous"] | r["ambiguous"]
        out.pop("raw")
        for j, key in enumerate(("dfeatures", "dfeatures_abs", "dfeatures_maha", "dfeatures_amb")):
            out[key] = dfeat[j][:, :D]
        return out
    du = np.zeros((N, 1, 2)); dc = np.zeros((N, 1, 3)); da = np.zeros((N, 1, 1))
    dfeat = np.zeros((N, len(dl_t) * 3))
    amb = np.zeros(N, bool)
    for k, (trip, g) in enumerate(zip(_triples(f.astype(np.float64), D), dl_t)):
        r = orc.splat_backward(height, width, us, cinv2ds, alphas, np.ascontiguousarray(trip, np.float32), fwd,
                               np.ascontiguousarray(np.moveaxis(g, -1, 0), np.float32), return_ambiguous=True,
                               margin=margin)
        du += r[0]; dc += r[1]; da += r[2]
        dfeat[:, 3 * k:3 * k + 3] = r[3].reshape(N, 3)
        amb |= r[4]
    out = (du, dc, da, dfeat[:, :D])
    return out + (amb,) if return_ambiguous else out


def step_features(scene, cam, *, aa, filt, features, dl, dF, drawn_inputs=None):
    """One GSFunctionFusedFeatures step in fp64: the colour step of `step_oracle.step` (rgbd and pose
    off) with the feature map's rasterizer gradients added before the chain.  features[N, D]; dl [3,H,W]
    and dF [D,H,W] (zeros for a map the loss does not use).  drawn_inputs: as for `step_oracle.step`.
    -> dict(image, features[D,H,W], ambiguous[H,W], thin_pixels, grads (pws, shs, scales, rots, alphas,
    us, features), flagged[N], thin[N], band[N])"""
    H, W = cam["height"], cam["width"]
    fw = ost.forward(scene, cam, aa=aa, filt=filt)
    st = fw["st"]
    N = len(fw["af"])
    inp = drawn_inputs if drawn_inputs is not None else dict(
        us=st["us"], ci=st["ci"], col=st["col"], depths=st["depths"], areas=st["areas"], alphas=fw["drawn"])
    out = ost.render(cam, False, inp)
    fout = splat_features(H, W, inp["us"], inp["ci"], inp["alphas"], inp["depths"], inp["areas"], features)
    du, dc, da, dcol, amb = orc.splat_backward(H, W, inp["us"], inp["ci"], inp["alphas"], inp["col"], out,
                                               np.asarray(dl, np.float32), return_ambiguous=True)
    fdu, fdc, fda, dfeat, famb = splat_backward_features(H, W, inp["us"], inp["ci"], inp["alphas"], out, features, dF,
                                                         return_ambiguous=True)
    du, dc, da, amb = du + fdu, dc + fdc, da + fda, amb | famb
    Rcw = cam["Rcw"]
    ch = orc.chain_backward(Rcw, du, dc, da, dcol, *st["J"])
    da_eff = da.reshape(N)
    g = dict(shs=ch["shs"], us=ch["us"].reshape(N, 2), features=dfeat)
    if aa:
        add = oaa.chain(st, Rcw, oaa.dcov2d_addend(st["c2"], st["keep"], fw["af"], da_eff))
        for k in ("pws", "scales", "rots"):
            g[k] = ch[k] + add[k]
    else:
        g.update(pws=ch["pws"], scales=ch["scales"], rots=ch["rots"])
    dalpha_f = fw["rho"] * da_eff if aa else da_eff
    if filt is None:
        g["alphas"] = dalpha_f
    else:
        g["scales"], g["alphas"] = of3.backward(scene["scales"], scene["alphas"], filt, g["scales"], dalpha_f)
    # the rows and pixels step_oracle.step flags, computed there (the colour step shares the forward)
    ref = ost.step(scene, cam, rgbd=False, pose=False, aa=aa, filt=filt, dl=np.zeros((3, H, W), np.float32),
                   drawn_inputs=drawn_inputs)
    return dict(image=out["image"], features=fout["features"], ambiguous=out["ambiguous"] | fout["ambiguous"],
                thin_pixels=ref["thin_pixels"], grads=g, flagged=ref["flagged"] | amb, thin=ref["thin"],
                band=ref["band"])
