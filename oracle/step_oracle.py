"""fp64 whole training step of the fused classes, every flag: RGB-D, camera pose, antialiasing, the 3D
filter.  TEST INFRASTRUCTURE ONLY.

A composition of the existing oracles with no derivative of its own:
    1. filter3d_oracle.apply                       s', alpha'        (pass-through without a filter)
    2. aa_oracle.stages / scale                    the stages on s'; alpha_eff = rho alpha' (AA) or alpha'
    3. oracle.splat or rgbd_oracle.splat_rgbd      image (D, A)
    4. splat_backward(_rgbd) -> oracle.chain_backward
       + aa_oracle.dcov2d_addend (alpha', dL/dalpha_eff) through aa_oracle.chain
       + rgbd_oracle.chain_depth
       camera: pose_oracle.camera_grad + aa_oracle.camera
       dL/dalpha' = rho dL/dalpha_eff, then filter3d_oracle.backward -> dL/ds, dL/dalpha
`flagged` marks the rows whose fp32 gradient may legitimately leave the strict bound (see `step`).
"""
import numpy as np

from . import aa_oracle as oaa
from . import filter3d_oracle as of3
from . import oracle as orc
from . import pose_oracle as opose
from . import rgbd_oracle as ordb

Z_BAND = 1e-5  # |z - 0.2| below this: the near-plane cull may go either way in fp32


def camera(sc, width, height):
    """the camera fields of a scene dict (Rcw, tcw, twc, fx, fy, cx, cy) and the frame size"""
    c = {k: sc[k] for k in ("Rcw", "tcw", "twc", "fx", "fy", "cx", "cy")}
    c.update(width=int(width), height=int(height))
    return c


def forward(scene, cam, *, aa, filt):
    """steps 1-2 -> dict(sf, af (s', alpha' in fp64), st (aa_oracle.stages on s'), scale (aa_oracle.scale),
    rho (1 without AA), drawn (the opacities the rasterizer composites))"""
    if filt is None:
        sf = np.asarray(scene["scales"], np.float64).reshape(-1, 3)
        af = np.asarray(scene["alphas"], np.float64).reshape(-1)
    else:
        sf, af, _ = of3.apply(scene["scales"], scene["alphas"], filt)
    st = oaa.stages(scene["pws"], scene["rots"], sf, scene["shs"], cam["Rcw"], cam["tcw"], cam["twc"], cam["fx"],
                    cam["fy"], cam["cx"], cam["cy"], cam["width"], cam["height"])
    s = oaa.scale(st["c2"], st["keep"])
    rho = s["rho"] if aa else np.ones(len(af))
    return dict(sf=sf, af=af, st=st, scale=s, rho=rho, drawn=rho * af)


def render(cam, rgbd, inp):
    """step 3 on inp = dict(us, ci, col, depths, areas, alphas) (copied: the binning culls in place)"""
    H, W = cam["height"], cam["width"]
    d = np.array(inp["depths"], np.float32).reshape(-1)
    ar = np.array(inp["areas"], np.int32)
    draw = ordb.splat_rgbd if rgbd else orc.splat
    return draw(H, W, inp["us"], inp["ci"], inp["alphas"], d, inp["col"], ar)


def loss(out, dl, dld=None, dla=None):
    """L = <dl, image> + <dld, D> + <dla, A> of a `render` result"""
    val = float((out["image"] * dl).sum())
    if dld is not None:
        val += float((out["depth"] * dld).sum())
    if dla is not None:
        val += float((out["alpha"] * dla).sum())
    return val


def step(scene, cam, *, rgbd, pose, aa, filt, dl, dld=None, dla=None, drawn_inputs=None):
    """One fused training step in fp64.  scene: dict(pws, rots, scales, shs, alphas) (fp32 arrays);
    cam: `camera(...)`; filt: None or the filter[N]; dl[3,H,W] (dld, dla [H,W]: the RGB-D planes'
    upstream gradients, 0 when None).  drawn_inputs: None (render on the oracle's own stage outputs) or
    dict(us, ci, col, depths, areas, alphas) -- the kernel's fp32 values, so that the rasterizer's
    threshold decisions are taken on the values the device composited.
    -> dict(image, depth, alpha (None without rgbd), ambiguous[H,W], thin_pixels[H,W] (the footprints of
    the thin rows), grads (pws, shs, scales, rots, alphas, us), raster (du, dc, da, dcol, dz), per[N,15] and
    absum[15] (zeros without pose), cam_grad, flagged[N], thin[N], band[N], fwd (forward's dict))
    flagged: rasterizer-ambiguous rows, the near-plane band, aa_oracle.thin rows (on s'), and with AA the
    rows aa_oracle.flagged marks."""
    H, W = cam["height"], cam["width"]
    fw = forward(scene, cam, aa=aa, filt=filt)
    st, s = fw["st"], fw["scale"]
    N = len(fw["af"])
    inp = drawn_inputs if drawn_inputs is not None else dict(
        us=st["us"], ci=st["ci"], col=st["col"], depths=st["depths"], areas=st["areas"], alphas=fw["drawn"])
    out = render(cam, rgbd, inp)
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
    gc2 = oaa.dcov2d_addend(st["c2"], st["keep"], fw["af"], da_eff) if aa else np.zeros((N, 3))
    g = dict(shs=ch["shs"], us=ch["us"].reshape(N, 2))
    if aa:
        add = oaa.chain(st, Rcw, gc2)
        for k in ("pws", "scales", "rots"):
            g[k] = ch[k] + add[k]
    else:
        g.update(pws=ch["pws"], scales=ch["scales"], rots=ch["rots"])
    if rgbd:
        g["pws"] = g["pws"] + ordb.chain_depth(Rcw, dz, st["depths"])
    dalpha_f = fw["rho"] * da_eff if aa else da_eff
    if filt is None:
        g["alphas"] = dalpha_f
    else:
        g["scales"], g["alphas"] = of3.backward(scene["scales"], scene["alphas"], filt, g["scales"], dalpha_f)
    if pose:
        per = opose.camera_grad(st, scene["pws"], Rcw, cam["fx"], cam["fy"], W, H, du, dc, dcol, dz)["per"]
        if aa:
            per = per + oaa.camera(st, scene["pws"], Rcw, cam["fx"], cam["fy"], W, H, gc2)
    else:
        per = np.zeros((N, 15))
    R64 = np.asarray(Rcw, np.float32).astype(np.float64).reshape(3, 3)
    z64 = np.asarray(scene["pws"], np.float32).astype(np.float64) @ R64[2] + float(np.float32(cam["tcw"][2]))
    band = np.abs(z64 - 0.2) < Z_BAND
    thin = oaa.thin(fw["sf"])
    flagged = amb | band | thin
    if aa:
        flagged = flagged | oaa.flagged(fw["sf"], s)
    # the pixels a thin row composites into (alpha' >= 0.001, half the skip threshold): an fp32 conic that
    # long evaluates the exponent with an absolute error of ~2^-24 (|a| dx^2 + 2 |b dx dy| + |c| dy^2),
    # far above the pixel tolerance.  (A row composites anywhere in the 16x16 tiles its rectangle touches.)
    foot = np.zeros((H, W), bool)
    us, areas = np.asarray(inp["us"], np.float64).reshape(N, 2), np.asarray(inp["areas"]).reshape(N, 2)
    ci, al = np.asarray(inp["ci"], np.float64).reshape(N, 3), np.asarray(inp["alphas"], np.float64).reshape(N)
    for i in np.flatnonzero(thin & (areas.max(1) > 0) & (al > 0)):
        (u, v), (ax, ay) = us[i], areas[i]
        y0, y1 = max(0, int(v - ay) // 16 * 16), min(H, (int(v + ay) // 16 + 1) * 16)
        x0, x1 = max(0, int(u - ax) // 16 * 16), min(W, (int(u + ax) // 16 + 1) * 16)
        if y0 >= y1 or x0 >= x1:
            continue
        dy, dx = np.mgrid[y0:y1, x0:x1].astype(np.float64)
        dx, dy = dx - u, dy - v
        p = -0.5 * (ci[i, 0] * dx * dx + ci[i, 2] * dy * dy) - ci[i, 1] * dx * dy
        foot[y0:y1, x0:x1] |= al[i] * np.exp(np.minimum(p, 0.0)) >= 1e-3
    return dict(image=out["image"], depth=out.get("depth"), alpha=out.get("alpha"), ambiguous=out["ambiguous"],
                thin_pixels=foot, grads=g, raster=(du, dc, da, dcol, dz), per=per, absum=np.abs(per).sum(0),
                cam_grad=per.sum(0), flagged=flagged, thin=thin, band=band, fwd=fw)
