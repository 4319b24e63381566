"""CPU checks of the oracle's per-entry moment rows and their conditioning (`oracle.drawB_rows`), the
reference tests/test_gpu_raster_rows.py holds the backward rasterizers to, entry by entry:

- converted with k_finalize_grads' formulas, the rows are orc_drawB's gradients (orc_drawB_rgbd's with
  the RGB-D channels, orc_drawB_abs's signed and absolute sums) to 1e-12, on the parity frames and the
  edge scenes;
- abs_rows >= |rows| everywhere, with equality for a one-pixel Gaussian and a scene whose terms all have
  one sign; drawn Gaussians none of whose pixels composite have exact zeros in every row;
- amb_rows = 0 at margin 0;
- the feature oracle's triple sums equal one all-channel run, for D in {1, 3, 4, 17}.
The oracle runs on one OpenMP thread wherever bits are compared: its sums use `omp atomic` under a
dynamic schedule."""
import numpy as np
import pytest

from oracle import absgrad_oracle as oabs
from oracle import feature_oracle as ofe
from oracle import oracle as orc
from oracle import rgbd_oracle as orgbd
from easygaussiansplatting_b200.scene import upstream_gradient

from test_gpu_parity import (boundary_frame, boundary_scene, clamp_scene, dense_scene, huge_needle_scene,
                             scene_with_culls)
from test_rgbd_edge_scenes_cpu import part_inputs, scene_inputs


@pytest.fixture(autouse=True)
def one_thread():
    n0 = orc.num_threads()
    orc.set_num_threads(1)
    yield
    orc.set_num_threads(n0)


def case(name):
    """-> (H, W, (us, cinv2ds, alphas, depths, colors, areas) fp32, seed)"""
    if name == "boundary":
        parts, expect, _, _ = boundary_scene(np.random.default_rng(7))
        W, H = boundary_frame(expect)
        return H, W, part_inputs(parts), 7
    if name.startswith("frame"):
        N, W, H = (int(x) for x in name.split("_")[1:])
        sc, seed = scene_with_culls(N, W, H, 3, N), N
    else:
        sc, seed = {"dense": (dense_scene(), 11), "clamp": (clamp_scene(), 2), "huge_needle": (huge_needle_scene(), 13)}[name]
    return sc["height"], sc["width"], scene_inputs(sc), seed


CASES = ["frame_3000_250_130", "frame_10000_256_256", "frame_3000_979_546", "frame_40_17_9", "boundary", "dense",
         "clamp", "huge_needle"]


def close(a, b, what, rel=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64).reshape(np.shape(a))
    s = max(float(np.abs(b).max(initial=0.0)), 1e-300)
    assert float(np.abs(a - b).max(initial=0.0)) <= rel * s, what


def covers(ab, rows, what):
    assert (ab >= np.abs(rows) * (1 - 1e-12)).all(), what


@pytest.mark.parametrize("name", CASES)
def test_rows_convert_to_drawB_and_bound_their_values(name):
    H, W, (us, ci, al, d, col, ar), seed = case(name)
    fwd = orc.splat(H, W, us, ci, al, d.copy(), col, ar.copy())
    dl = upstream_gradient(W, H, seed) * np.float32(3.0 * W * H)
    r = oabs.splat_backward_abs_rows(H, W, us, ci, al, col, fwd, dl)
    *want, amb = orc.splat_backward(H, W, us, ci, al, col, fwd, dl, return_ambiguous=True)
    for got, w, what in zip(orc.moments_to_grads(r["rows"], ci), want, ("dus", "dcinv2ds", "dalphas", "dcolors")):
        close(got, w, what)
    assert np.array_equal(r["ambiguous"], amb)
    du, dabs, _ = oabs.splat_backward_abs(H, W, us, ci, al, col, fwd, dl)
    close(r["dus_abs"], dabs, "dus_abs")
    covers(r["abs_rows"], r["rows"], "abs_rows")
    covers(r["dus_abs_abs"], r["dus_abs"], "dus_abs_abs")
    for k in ("maha_rows", "amb_rows"):
        assert (r[k] >= 0).all() and np.isfinite(r[k]).all(), k
    # the conditioning carried through the conversion bounds the converted values
    for got, b in zip(orc.moments_to_grads(r["rows"], ci), orc.moments_to_grads_bound(r["abs_rows"], ci)):
        covers(b, got, "converted abs rows")
    # drawn Gaussians none of whose pixels composite: exact zeros in every row
    drawn = np.zeros(len(us), bool)
    drawn[fwd["gsid"]] = True
    quiet = drawn & ~r["abs_rows"].any(axis=1) & ~r["amb_rows"].any(axis=1)
    assert not r["rows"][quiet].any() and not r["maha_rows"][quiet].any() and not r["dus_abs"][quiet].any()
    if name == "clamp":  # rows of opacity 0.001 never composite
        assert quiet.sum() >= (al[drawn] == np.float32(0.001)).sum() > 0
    # margin 0: nothing is ambiguous
    r0 = oabs.splat_backward_abs_rows(H, W, us, ci, al, col, fwd, dl, margin=0.0)
    assert not r0["amb_rows"].any() and not r0["dus_abs_amb"].any()
    assert np.array_equal(r0["rows"], r["rows"]) and np.array_equal(r0["abs_rows"], r["abs_rows"])


@pytest.mark.parametrize("name", ["frame_3000_250_130", "boundary", "dense", "clamp", "huge_needle"])
def test_rgbd_rows_convert_to_drawB_rgbd(name):
    H, W, (us, ci, al, d, col, ar), seed = case(name)
    fwd = orgbd.splat_rgbd(H, W, us, ci, al, d.copy(), col, ar.copy())
    rng = np.random.default_rng(seed)
    dl = upstream_gradient(W, H, seed) * np.float32(3.0 * W * H)
    dld, dla = (rng.normal(size=(H, W)).astype(np.float32) for _ in range(2))
    for use in ((1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 1)):
        a, b, c = (x if u else np.zeros_like(x) for x, u in zip((dl, dld, dla), use))
        r = oabs.splat_backward_abs_rows(H, W, us, ci, al, col, fwd, a, depths=fwd["z"], dloss_ddepth=b, dloss_dalpha=c)
        want = orgbd.splat_backward_rgbd(H, W, us, ci, al, col, fwd["z"], fwd, a, b, c)
        for got, w, what in zip(orc.moments_to_grads(r["rows"], ci) + (r["ddepths"],), want,
                                ("dus", "dcinv2ds", "dalphas", "dcolors", "ddepths")):
            close(got, w, "%s %s" % (what, use))
        _, dabs, _ = oabs.splat_backward_rgbd_abs(H, W, us, ci, al, col, fwd["z"], fwd, a, b, c)
        close(r["dus_abs"], dabs, "dus_abs %s" % (use,))
        covers(r["abs_rows"], r["rows"], "abs_rows")
        covers(r["ddepths_abs"], r["ddepths"], "ddepths_abs")
        if use == (0, 0, 1):  # dL/dA alone: no colour and no depth term
            assert not r["rows"][:, 6:].any() and not r["ddepths"].any()
    # with dL/dD = dL/dA = 0 the RGB-D rows are the colour rows
    z = np.zeros((H, W), np.float32)
    rc = orc.splat_backward_rows(H, W, us, ci, al, col, fwd, dl)
    r = orgbd.splat_backward_rgbd_rows(H, W, us, ci, al, col, fwd["z"], fwd, dl, z, z)
    for k in ("rows", "abs_rows", "maha_rows", "amb_rows"):
        close(r[k], rc[k], k, rel=1e-15)


def one_gaussian(alpha, sigma, u, H=16, W=16):
    us = np.array([u], np.float32)
    ci = np.array([[1 / sigma ** 2, 0.0, 1 / sigma ** 2]], np.float32)
    return us, ci, np.array([alpha], np.float32), np.array([1.0], np.float32), np.array([[0.8, 0.5, 0.2]], np.float32), \
        np.array([[2, 2]], np.int32)


def test_one_pixel_gaussian_and_one_sign_terms_are_their_own_conditioning():
    H = W = 16
    # a Gaussian that composites exactly one pixel: every entry is a single product
    us, ci, al, d, col, ar = one_gaussian(0.9, 0.2, (5.05, 6.1))
    fwd = orc.splat(H, W, us, ci, al, d.copy(), col, ar.copy())
    assert (fwd["contrib"] > 0).sum() == 1
    dl = np.abs(np.random.default_rng(1).normal(size=(3, H, W))).astype(np.float32)  # one sign per product
    r = oabs.splat_backward_abs_rows(H, W, us, ci, al, col, fwd, dl)
    close(r["abs_rows"], np.abs(r["rows"]), "one pixel", rel=1e-15)
    # one Gaussian under positive dL/dgamma and colours, centred on a pixel corner (dx, dy > 0 on its pixels
    # left of and above the centre): w > 0 and every moment of the quarter-plane has one sign
    us, ci, al, d, col, ar = one_gaussian(0.5, 2.0, (10.0, 10.0))
    fwd = orc.splat(H, W, us, ci, al, d.copy(), col, ar.copy())
    dl = np.zeros((3, H, W), np.float32)
    dl[:, :10, :10] = 1.0  # pixels with dx, dy >= 1 only
    r = oabs.splat_backward_abs_rows(H, W, us, ci, al, col, fwd, dl)
    assert (r["rows"] > 0).all()
    close(r["abs_rows"], r["rows"], "one sign", rel=1e-15)
    close(r["dus_abs_abs"], r["dus_abs"], "one sign, AbsGS", rel=1e-15)


@pytest.mark.parametrize("D", [1, 3, 4, 17])
def test_feature_triples_sum_to_one_all_channel_run(D):
    H, W, (us, ci, al, d, col, ar), seed = case("frame_3000_250_130")
    fwd = orc.splat(H, W, us, ci, al, d.copy(), col, ar.copy())
    rng = np.random.default_rng(D)
    f = rng.normal(size=(len(us), D)).astype(np.float32)
    dF = rng.normal(size=(D, H, W)).astype(np.float32)
    trip = ofe.splat_backward_features(H, W, us, ci, al, fwd, f, dF, rows=True)
    R, Ab, Mh, Am, amb = orc.drawB_rows(H, W, us, ci, al, f, fwd, dF)
    for key, a in zip(("rows", "abs_rows", "maha_rows", "amb_rows"), (R, Ab, Mh, Am)):
        close(trip[key][:, :6], a[:, :6], key)
        assert not trip[key][:, 6:].any()
    for key, a in zip(("dfeatures", "dfeatures_abs", "dfeatures_maha", "dfeatures_amb"), (R, Ab, Mh, Am)):
        close(trip[key], a[:, 8:], key)
    assert np.array_equal(trip["ambiguous"], amb)
    # and the signed sums are splat_backward_features'
    want = ofe.splat_backward_features(H, W, us, ci, al, fwd, f, dF)
    for got, w, what in zip(orc.moments_to_grads(np.concatenate([trip["rows"][:, :6], np.zeros((len(us), 3))], 1),
                                                 ci)[:3] + (trip["dfeatures"],), want,
                            ("dus", "dcinv2ds", "dalphas", "dfeatures")):
        close(got, w, what)
