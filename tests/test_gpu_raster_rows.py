"""The backward rasterizers per Gaussian entry against each entry's own fp64 conditioning.

Every output of k_draw_bwd, k_draw_bwd_rgbd, their AbsGS forms and k_draw_feat_bwd is a per-Gaussian sum
of per-pixel terms.  The per-tensor checks elsewhere hold an entry only to 1e-4 of the tensor's largest
one, so a small entry (deep in a stack, a faint tail, a few pixels at an odd edge) could be zeroed
unnoticed.  Here every entry e of every Gaussian, on the kernel's own fp32 inputs, must satisfy

    |got - ref| <= C_ABS abs_rows + C_MAHA maha_rows + amb_rows,    got == 0 where abs_rows = amb_rows = 0

with the oracle's rows (`oracle.drawB_rows`, gs_oracle.c): abs_rows sums the magnitudes of every product
in a term before any cancellation, maha_rows the terms' sensitivity to the exponents' rounding (it is
what needles cancel), amb_rows what a threshold decision within the oracle's margin can move (0 for
all but a few Gaussians).  The moment rows `splatB(..., moments_only=True)` returns are checked, and the
converted tensors of the full call with the conditioning carried through k_finalize_grads' formulas.
Flagged Gaussians (an alpha' in the skip window) stay under 1 % of the drawn ones.  C_ABS and C_MAHA
hold for all four kernels and every scene; the worst measured ratios are in DESIGN section 4.
"""
import numpy as np
import pytest
import torch

from oracle import absgrad_oracle as oabs
from oracle import feature_oracle as ofe
from oracle import oracle as orc
from oracle import rgbd_oracle as orgbd
from easygaussiansplatting_b200.scene import synthetic_scene, upstream_gradient

from test_gpu_parity import (DEV, boundary_frame, boundary_scene, clamp_scene, dead_sparse_scene, dense_scene,
                             huge_needle_scene, n, op_inputs, scene_with_culls, stage_pipeline, t)

pytestmark = pytest.mark.gpu

C_ABS = 2.0 ** -14  # 6.1e-6: 16x tighter than the surfel path's 1e-4
C_MAHA = 4 * 2.0 ** -24
WORST = {}  # (kernel, scene) -> worst err / (C_ABS abs + C_MAHA maha) over unflagged entries


def ops():
    from easygaussiansplatting_b200 import ops as o
    return o


@pytest.fixture(scope="module", autouse=True)
def report_worst_ratios():
    yield
    for (kernel, scene), r in sorted(WORST.items()):
        print("worst ratio %-12s %-22s %.3e" % (kernel, scene, r))


def check(got, want, ab, mh, am, kernel, scene, what):
    """the per-entry bound; records the worst unflagged ratio under (kernel, scene)"""
    want = np.asarray(want, np.float64)
    got = n(got).astype(np.float64).reshape(want.shape) if isinstance(got, torch.Tensor) else \
        np.asarray(got, np.float64).reshape(want.shape)
    assert np.isfinite(got).all(), what
    ab, mh, am = (np.asarray(x, np.float64).reshape(want.shape) for x in (ab, mh, am))
    dead = (ab == 0) & (am == 0)
    assert not got[dead].any(), "%s: %d entries without a term are not 0" % (what, int((got[dead] != 0).sum()))
    err = np.abs(got - want)
    cond = C_ABS * ab + C_MAHA * mh
    excess = err - cond - am
    i = np.unravel_index(np.argmax(excess), excess.shape) if excess.size else None
    assert excess.size == 0 or excess[i] <= 0, "%s: entry %s got %r want %r (abs %.3g maha %.3g amb %.3g)" % (
        what, i, got[i], want[i], ab[i], mh[i], am[i])
    live = (am == 0) & (cond > 0)
    r = float((err[live] / cond[live]).max(initial=0.0))
    WORST[(kernel, scene)] = max(WORST.get((kernel, scene), 0.0), r)
    return r


def check_flagged(ref, gsid):
    drawn = np.zeros(len(ref["ambiguous"]), bool)
    drawn[gsid] = True
    assert ref["ambiguous"][drawn].sum() <= 0.01 * max(drawn.sum(), 1), "flagged: %d of %d drawn" % (
        ref["ambiguous"][drawn].sum(), drawn.sum())


def check_moments(mom, ref, kernel, scene):
    """the moment rows [N,9] a kernel writes, before k_finalize_grads"""
    check(mom, ref["rows"], ref["abs_rows"], ref["maha_rows"], ref["amb_rows"], kernel, scene, kernel + " rows")


def check_converted(grads, ref, ci, kernel, scene):
    """what the full call returns: k_finalize_grads' formulas on the rows, the conditioning carried through them"""
    want = orc.moments_to_grads(ref["rows"], ci)
    cond = [orc.moments_to_grads_bound(ref[k], ci) for k in ("abs_rows", "maha_rows", "amb_rows")]
    for j, name in enumerate(("dus", "dcinv2ds", "dalphas", "dcolors")):
        check(grads[j], want[j], cond[0][j], cond[1][j], cond[2][j], kernel, scene, kernel + " " + name)


# ---------------------------------------------------------------- scenes (op-surface inputs)
PARITY_FRAMES = [(10000, 256, 256), (3000, 250, 130), (50000, 512, 512), (4001, 320, 200), (200, 64, 48),
                 (3000, 979, 546), (2000, 255, 131), (40, 17, 9), (8, 7, 5)]


def scene_inputs(name):
    """-> (H, W, us, cinv2ds, alphas, depths, colors, areas) device tensors of a scene, seed"""
    if name.startswith("frame"):
        N, W, H = (int(x) for x in name.split("_")[1:])
        sc = scene_with_culls(N, W, H, 3, N)
        seed = N
    elif name == "boundary":
        parts, expect, _, _ = boundary_scene(np.random.default_rng(7))
        W, H = boundary_frame(expect)
        return (H, W) + op_inputs(parts), 7
    elif name == "dead4k":
        parts = dead_sparse_scene(np.random.default_rng(11))
        return (2160, 3840) + op_inputs(parts), 11
    else:
        sc, seed = {"dense": (dense_scene(), 11), "clamp": (clamp_scene(), 2), "huge_needle": (huge_needle_scene(), 13)}[name]
    o = stage_pipeline(sc, calc_J=False)
    return (sc["height"], sc["width"], o["us"], o["cinv2ds"], t(sc["alphas"]), o["depths"], o["colors"],
            o["areas"]), seed


SCENES = ["frame_%d_%d_%d" % f for f in PARITY_FRAMES] + ["boundary", "dense", "clamp", "huge_needle", "dead4k"]


def draw(H, W, us, ci, al, d, col, ar, rgbd=False, capacity=False, records=None):
    """ops.splat(_rgbd) on copies of depths / areas, and the oracle's forward on the same fp32 values"""
    o = ops()
    h = [n(x) for x in (us, ci, al, col)]
    d_in, a_in = n(d).copy(), n(ar).copy()
    d1, a1 = d.clone(), ar.clone()
    if rgbd:
        out = o.splat_rgbd(H, W, us, ci, al, d1, col, a1, capacity=capacity, records=records)
        ref = orgbd.splat_rgbd(H, W, *h[:3], d_in.copy(), h[3], a_in.copy())
    else:
        out = o.splat(H, W, us, ci, al, d1, col, a1, capacity=capacity, records=records)
        ref = orc.splat(H, W, *h[:3], d_in.copy(), h[3], a_in.copy())
    assert np.array_equal(n(out[4]), ref["gsid"]) and np.array_equal(n(out[3]), ref["ranges"])
    return out, ref, h, d1


# ---------------------------------------------------------------- k_draw_bwd, k_draw_bwd_abs
def colour_case(H, W, us, ci, al, d, col, ar, seed, scene, capacity=False, records=None, repack=False):
    o = ops()
    out, fwd, (h_us, h_ci, h_al, h_col), d1 = draw(H, W, us, ci, al, d, col, ar, capacity=capacity, records=records)
    if repack:
        o.forget_records(out[4])
    dl = upstream_gradient(W, H, seed) * (3.0 * W * H)
    ref = oabs.splat_backward_abs_rows(H, W, h_us, h_ci, h_al, h_col, fwd, dl)
    check_flagged(ref, fwd["gsid"])
    args = (H, W, us, ci, al, d1, col, *out[1:5], t(dl))
    mom = o.splatB(*args, moments_only=True, records=records)
    check_moments(mom, ref, "k_draw_bwd", scene)
    check_converted(o.splatB(*args, records=records), ref, h_ci, "k_draw_bwd", scene)
    mom_a, dabs = o.splatB(*args, moments_only=True, records=records, absgrad=True)
    check_moments(mom_a, ref, "k_draw_bwd_abs", scene)
    check(dabs, ref["dus_abs"], ref["dus_abs_abs"], ref["dus_abs_maha"], ref["dus_abs_amb"], "k_draw_bwd_abs", scene,
          "dus_abs")
    return ref


@pytest.mark.parametrize("scene", SCENES)
def test_colour_rows_per_entry(scene):
    inp, seed = scene_inputs(scene)
    colour_case(*inp, seed, scene)


def test_colour_rows_capacity_path_and_records_given_and_repacked():
    """the capacity path, records from `preprocess` and records re-packed by splatB, at 979x546"""
    o = ops()
    N, W, H = 3000, 979, 546
    sc = scene_with_culls(N, W, H, 12, 21)
    p = {k: t(sc[k]) for k in ("pws", "rots", "scales", "shs", "Rcw", "tcw", "twc")}
    al = t(sc["alphas"])
    us, ci, col, d, ar, rec = o.preprocess(p["pws"], p["rots"], p["scales"], p["shs"], p["Rcw"], p["tcw"], p["twc"],
                                           sc["fx"], sc["fy"], sc["cx"], sc["cy"], W, H, alphas=al)
    o._CAPACITY.pop((torch.device(DEV).index or 0, H, W, N), None)
    for kw in (dict(capacity=True), dict(capacity=True), dict(records=rec), dict(repack=True)):
        colour_case(H, W, us, ci, al, d, col, ar, 21, "paths_979x546", **kw)


def test_colour_rows_config2_frame():
    """1M Gaussians at 1920x1080, SH degree 3 (BASELINE config 2)"""
    N, W, H = 1_000_000, 1920, 1080
    sc = synthetic_scene(N, W, H, sh_dim=48, seed=0)
    o = stage_pipeline(sc, calc_J=False)
    colour_case(H, W, o["us"], o["cinv2ds"], t(sc["alphas"]), o["depths"], o["colors"], o["areas"], 0, "config2")


# ---------------------------------------------------------------- k_draw_bwd_rgbd, k_draw_bwd_rgbd_abs
def upstream_planes(W, H, seed, zmax):
    rng = np.random.default_rng(seed + 101)
    dl = upstream_gradient(W, H, seed) * (3.0 * W * H)
    dld = (rng.normal(size=(H, W)) / zmax).astype(np.float32)
    dla = rng.normal(size=(H, W)).astype(np.float32)
    return dl, dld, dla


@pytest.mark.parametrize("scene", SCENES)
def test_rgbd_rows_per_entry(scene):
    """each of dL/dgamma, dL/dD, dL/dA alone and all three, moment rows, dL/dz and the converted tensors; the
    _abs form on all three"""
    o = ops()
    (H, W, us, ci, al, d, col, ar), seed = scene_inputs(scene)
    out, fwd, (h_us, h_ci, h_al, h_col), d1 = draw(H, W, us, ci, al, d, col, ar, rgbd=True)
    z = fwd["z"]
    zmax = max(float(np.abs(z[fwd["gsid"]]).max(initial=0.0)), 1.0)
    full = upstream_planes(W, H, seed, zmax)
    for use in ((1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 1)):
        dl, dld, dla = (x if u else np.zeros_like(x) for x, u in zip(full, use))
        ref = oabs.splat_backward_abs_rows(H, W, h_us, h_ci, h_al, h_col, fwd, dl, depths=z, dloss_ddepth=dld,
                                           dloss_dalpha=dla)
        check_flagged(ref, fwd["gsid"])
        args = (H, W, us, ci, al, d1, col, *out[1:5], t(dl), t(dld), t(dla))
        mom, dz = o.splatB_rgbd(*args, moments_only=True)
        check_moments(mom, ref, "k_draw_bwd_rgbd", scene)
        check(dz, ref["ddepths"], ref["ddepths_abs"], ref["ddepths_maha"], ref["ddepths_amb"], "k_draw_bwd_rgbd",
              scene, "ddepths %s" % (use,))
        g = o.splatB_rgbd(*args)
        check_converted(g, ref, h_ci, "k_draw_bwd_rgbd", scene)
        check(g[4], ref["ddepths"], ref["ddepths_abs"], ref["ddepths_maha"], ref["ddepths_amb"], "k_draw_bwd_rgbd",
              scene, "ddepths (full call) %s" % (use,))
        if use == (1, 1, 1):
            mom_a, dz_a, dabs = o.splatB_rgbd(*args, moments_only=True, absgrad=True)
            check_moments(mom_a, ref, "k_draw_bwd_rgbd_abs", scene)
            check(dz_a, ref["ddepths"], ref["ddepths_abs"], ref["ddepths_maha"], ref["ddepths_amb"],
                  "k_draw_bwd_rgbd_abs", scene, "ddepths")
            check(dabs, ref["dus_abs"], ref["dus_abs_abs"], ref["dus_abs_maha"], ref["dus_abs_amb"],
                  "k_draw_bwd_rgbd_abs", scene, "dus_abs")


# ---------------------------------------------------------------- k_draw_feat_bwd
FEATURE_WIDTHS = [1, 3, 4, 5, 6, 7, 8, 9, 12, 13, 16, 17, 33]


@pytest.mark.parametrize("scene", ["frame_2000_255_131", "frame_3000_979_546", "boundary", "clamp", "huge_needle"])
@pytest.mark.parametrize("D", FEATURE_WIDTHS)
def test_feature_rows_per_entry(scene, D):
    """every D mod 8 and both last-group widths; the moment rows on top of the colour rows (moments=)"""
    o = ops()
    (H, W, us, ci, al, d, col, ar), seed = scene_inputs(scene)
    out, fwd, (h_us, h_ci, h_al, h_col), d1 = draw(H, W, us, ci, al, d, col, ar)
    N = h_us.shape[0]
    f = np.random.default_rng(seed + D).normal(size=(N, D)).astype(np.float32)
    dF = np.random.default_rng(seed + 5 + D).normal(size=(D, H, W)).astype(np.float32)
    ref = ofe.splat_backward_features(H, W, h_us, h_ci, h_al, fwd, f, dF, rows=True)
    check_flagged(ref, fwd["gsid"])
    kw = dict(us=us, cinv2ds=ci, alphas=al, colors=col)
    mom, dfeat = o.splatB_features(H, W, t(f), out[1], out[2], out[3], out[4], t(dF), **kw)
    check_moments(mom, ref, "k_draw_feat_bwd", scene)
    check(dfeat, ref["dfeatures"], ref["dfeatures_abs"], ref["dfeatures_maha"], ref["dfeatures_amb"],
          "k_draw_feat_bwd", scene, "dfeatures D=%d" % D)
    if D in (3, 17):  # added to the colour rows
        dl = upstream_gradient(W, H, seed) * (3.0 * W * H)
        col_ref = orc.splat_backward_rows(H, W, h_us, h_ci, h_al, h_col, fwd, dl)
        base = o.splatB(H, W, us, ci, al, d1, col, *out[1:5], t(dl), moments_only=True)
        both, _ = o.splatB_features(H, W, t(f), out[1], out[2], out[3], out[4], t(dF), moments=base, **kw)
        summed = {k: col_ref[k] + ref[k] for k in ("rows", "abs_rows", "maha_rows", "amb_rows")}
        check_moments(both, summed, "k_draw_feat_bwd", scene)
