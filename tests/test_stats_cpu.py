"""CPU checks of the contribution statistics (DESIGN 3.18): the fp64 statistics oracles
(oracle/stats_oracle.py) against oracles already trusted -- the RGB-D oracle's alpha plane, the
feature oracle's dL/dfeatures for features = 1, dL/dF = 1, and a direct count of the (pixel, record)
pairs the colour oracle composites -- and the surfel statistics against surfel_oracle.render's alpha
plane; the C ABI of the new entry points and their profile ids."""
import ctypes as C

import numpy as np
import pytest

from oracle import feature_oracle as ofe
from oracle import oracle as orc
from oracle import rgbd_oracle as orgbd
from oracle import stats_oracle as ost
from oracle import surfel_oracle as so

from test_rgbd_cpu import _scene64, _stages

W, H, N = 97, 61, 600


def _frame(seed=3, n=N, w=W, h=H):
    sc = _scene64(n, w, h, seed=seed)
    us, ci, col, d32, areas, _ = _stages(sc, w, h)
    return sc, us, ci, col, d32, areas


def _composited_pairs(fwd, us, ci, al, w, h):
    """the (pixel, record) pairs the colour oracle composites, counted per Gaussian in numpy: the
    records before the pixel's contrib whose alpha' reaches 0.002"""
    us, ci, al = (np.asarray(a, np.float64) for a in (us, ci, al))
    al = al.reshape(-1)
    cnt = np.zeros(len(al), np.int64)
    gx = (w + 15) // 16
    for t, (s, e) in enumerate(fwd["ranges"]):
        if e <= s:
            continue
        ys, xs = np.mgrid[(t // gx) * 16:min((t // gx) * 16 + 16, h), (t % gx) * 16:min((t % gx) * 16 + 16, w)]
        xs, ys = xs.ravel(), ys.ravel()
        cont = fwd["contrib"][ys, xs]
        for j, g in enumerate(fwd["gsid"][s:e]):
            dx, dy = us[g, 0] - xs, us[g, 1] - ys
            m = np.maximum(ci[g, 0] * dx * dx + ci[g, 2] * dy * dy + 2 * ci[g, 1] * dx * dy, 0)
            ap = np.minimum(0.99, al[g] * np.exp(-0.5 * m))
            cnt[g] += int(((j < cont) & (ap >= 0.002)).sum())
    return cnt


@pytest.mark.parametrize("seed,n,w,h", [(3, N, W, H), (7, 2000, 64, 48), (11, 40, 17, 9)])
def test_colour_statistics_against_the_trusted_oracles(seed, n, w, h):
    sc, us, ci, col, d32, areas = _frame(seed, n, w, h)
    al = sc["alphas"]
    g = orgbd.splat_rgbd(h, w, us, ci, al, d32.copy(), col, areas.copy())
    st = ost.splat_stats(h, w, us, ci, al, g)
    # sum_i weight_sum_i = sum_p alpha(p)
    assert abs(st["weight_sum"].sum() - g["alpha"].sum()) <= 1e-12 * g["alpha"].sum()
    # weight_sum = dL/dfeatures for features = 1, dL/dF = 1
    ones = np.ones((n, 1), np.float32)
    df = ofe.splat_backward_features(h, w, us, ci, al, g, ones, np.ones((1, h, w), np.float32))[3]
    np.testing.assert_allclose(st["weight_sum"], df[:, 0], rtol=1e-12, atol=1e-15)
    # the counts are the composited pairs, the maxima at most the clamp, the sums at most the counts
    assert np.array_equal(st["hit_count"], _composited_pairs(g, us, ci, al, w, h))
    assert st["weight_max"].max() <= 0.99 and (st["weight_max"] <= st["weight_sum"] + 1e-15).all()
    assert (st["weight_sum"] <= st["hit_count"] * st["weight_max"] * (1 + 1e-12) + 1e-15).all()
    assert ((st["hit_count"] > 0) == (st["weight_sum"] > 0)).all()
    assert st["ambiguous"].mean() < 0.01


def test_a_gaussian_outside_every_tile_scores_zero():
    sc, us, ci, col, d32, areas = _frame(5)
    us = np.array(us, np.float32)
    us[:7] = (-500.0, -500.0)  # far outside the frame: no tile
    al = sc["alphas"]
    g = orc.splat(H, W, us, ci, al, d32.copy(), col, areas.copy())
    assert not np.isin(np.arange(7), g["gsid"]).any()
    st = ost.splat_stats(H, W, us, ci, al, g)
    for k in ("weight_sum", "weight_max", "hit_count"):
        assert not st[k][:7].any(), k
    assert st["hit_count"][7:].any()


def test_clamped_gaussians_peak_at_the_clamp():
    sc, us, ci, col, d32, areas = _frame(9)
    al = np.array(sc["alphas"], np.float32)
    al[:50] = 1.0  # alpha g > 0.99 near their centres
    g = orc.splat(H, W, us, ci, al, d32.copy(), col, areas.copy())
    st = ost.splat_stats(H, W, us, ci, al, g)
    assert st["weight_max"].max() == 0.99


def _surfel_scene(n, w, h, seed):
    rng = np.random.default_rng(seed)
    fx = fy = 0.8 * w
    zz = rng.uniform(2.0, 6.0, n)
    pws = np.stack([rng.uniform(-1, 1, n) * zz * w / (2 * fx), rng.uniform(-1, 1, n) * zz * h / (2 * fy), zz], 1)
    rots = rng.normal(size=(n, 4))
    scales = np.stack([rng.uniform(0.02, 0.15, n), rng.uniform(0.02, 0.15, n), rng.uniform(0.0, 0.05, n)], 1)
    shs = rng.normal(scale=0.3, size=(n, 3))
    alphas = rng.uniform(0.05, 0.95, n)
    alphas[:5] = 1.0
    f = lambda a: np.ascontiguousarray(a, dtype=np.float32)  # noqa: E731
    pre = so.preprocess(f(pws), f(rots), f(scales), f(shs), f(np.eye(3)), f(np.zeros(3)), f(np.zeros(3)), fx, fy,
                        w / 2 - 0.3, h / 2 + 0.2)
    return pre, f(alphas)


@pytest.mark.parametrize("n,w,h", [(300, 70, 45), (60, 33, 17)])
def test_surfel_statistics_against_the_surfel_oracle(n, w, h):
    pre, al = _surfel_scene(n, w, h, n)
    bins = so.bin_f32(h, w, pre)
    fwd = so.render(h, w, pre, al, bins)
    st = ost.surfel_stats(h, w, pre, al, bins)
    assert abs(st["weight_sum"].sum() - fwd["alpha"].sum()) <= 1e-12 * fwd["alpha"].sum()
    # the counts: per pixel, the records the walk composites (contrib - the skipped ones); in total the
    # pixels' composited records, recounted from the walk's own rule
    on = np.zeros(n, np.int64)
    alpha64 = al.astype(np.float64)
    for t, X, Y in so._tiles(h, w, bins[1]):
        tau = np.ones(len(X))
        for i in bins[2][bins[1][t, 0]:bins[1][t, 1]]:
            e = so._eval(pre["M"][i], pre["u"][i], X.astype(np.float64), Y.astype(np.float64))
            ap = np.minimum(0.99, alpha64[i] * np.exp(-0.5 * e["G"]))
            hit = (tau >= 1e-4) & (ap >= 0.002)
            on[i] += int(hit.sum())
            tau = np.where(hit, tau * (1 - ap), tau)
    assert np.array_equal(st["hit_count"], on)
    assert 0 < st["weight_max"].max() <= 0.99
    assert ((st["hit_count"] > 0) == (st["weight_sum"] > 0)).all()
    outside = ~np.isin(np.arange(n), bins[2])
    assert not st["hit_count"][outside].any()


def test_entry_points_and_profile_ids():
    from easygaussiansplatting_b200 import _lib
    lib = _lib.load()
    for name in ("gsb_splat_stats_workspace_bytes", "gsb_splat_stats", "gsb_splat_stats_2dgs",
                 "gsb_density_plan_keep"):
        assert name in _lib.SIGNATURES
        assert hasattr(lib, name)
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    i = names.index("draw_backward_features")
    assert names[i + 1:i + 4] == ["draw_stats", "draw_surfel_stats", "mcmc_scan"]
    # argument errors, before any device work
    counts = (C.c_int64 * 3)()
    assert lib.gsb_density_plan_keep(4, None, None, 0, None, None, counts, None) != 0
    assert b"density_plan_keep" in lib.gsb_last_error()
    assert lib.gsb_splat_stats_2dgs(0, 8, 1, 1, None, None, None, None, None, None, None, None) != 0
    assert b"bad N/H/W/P" in lib.gsb_last_error()
    buf = (C.c_char * 64)()
    base = C.addressof(buf)
    assert lib.gsb_splat_stats_2dgs(8, 8, 1, 1, None, None, None, None, base + 4, base + 8, base + 20, None) != 0
    assert b"misaligned output" in lib.gsb_last_error()
    assert lib.gsb_splat_stats_2dgs(8, 8, 1, 1, None, None, None, None, base, base + 8, base + 16, None) != 0
    assert b"null pointer" in lib.gsb_last_error()


def test_lowest_breaks_ties_by_index():
    import torch
    from easygaussiansplatting_b200.density import lowest
    s = torch.tensor([3.0, 1.0, 1.0, 2.0, 1.0, 0.5])
    keep = lowest(s, 0.5)  # drops 3 rows: 0.5, then the first two of the three 1.0
    assert keep.tolist() == [True, False, False, True, True, False]
    assert lowest(s, 0.0).all() and not lowest(s, 1.0).any()
    assert int((~lowest(torch.arange(10.0), 0.66)).sum()) == 6
    with pytest.raises(ValueError):
        lowest(s, 1.5)
