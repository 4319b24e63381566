"""2DGS geometry-term edge scenes (DESIGN 3.16), checked without a GPU.

The scene generators of tests/test_gpu_surfel_geometry_edges.py, each checked with the fp64 model
(tests/surfel_geometry_oracle.py) alone to reach the edge it is named for, and the model's own
claims on the surfel edge scenes of tests/test_surfel_edge_scenes_cpu.py.

Exact scenes.  At the identity camera with cx = cy = 0 and a power-of-two focal length F, a
fronto-parallel disk whose camera-frame centre is (x Z / F, y Z / F, Z) for an integer pixel (x, y)
and a depth Z = c / 2048 has every product the kernels form there exact in fp32: pc = pw, M's third
column is (F X, F Y, Z), the ray-plane cross terms x Z - F X vanish, so the plane point is (0, 0),
G3 = 0, the Gaussian factor ex2(0) = 1 and alpha' = alpha.  Every hit depth of a fronto-parallel
disk is its Z.  With alphas 0.5, 0.75 and 0.25 the transmittance products are exact too, so fp32
and fp64 see an incoming tau of exactly 0.5 and a hit exactly at `near` alike: the model reports
those pixels (render_geometry(exact=True)) instead of flagging them.  (At such a centre G3 = G2 = 0
and surfel_oracle flags the branch G3 <= G2; both sides take G3 there, and z and alpha' are the same
in either branch.)
"""
import numpy as np
import pytest

from oracle import surfel_oracle as so
import surfel_geometry_oracle as sg
from test_gpu_surfel_edges import with_culled
from test_surfel_edge_scenes_cpu import (dead_claims, dead_scene, dense_scene, fronto, margins, oracle_frame, place,
                                         pre_of, random_scene, special_scene, stack_scene)

F = 32.0


def dyadic_depths(z0, n):
    """n consecutive depths c / 2048 from about z0 whose millimetre depth keys floor(1000 z) all lie at
    least 0.01 from an integer (the margin of an exact independent binning)"""
    c = int(np.ceil(z0 * 2048))
    while True:
        z = (c + np.arange(n)) / 2048.0
        fr = z * 1000 - np.floor(z * 1000)
        if fr.min() >= 0.01 and fr.max() <= 0.99:
            return z
        c += 1


def exact_stacks(tiles, W, H, seed, k=1):
    """one list per tile of (alpha, at_centre, z): at_centre disks (sigma 2.2 px) centred exactly on
    the tile's pixel (8, 8), the others (fillers, sigma 0.8 px) at a tile corner 5.2 px away, where they
    composite without reaching the centre (alpha' < 1e-10 there).  Each list stays in its tile.
    Identity camera, cx = cy = 0, focal length F.  -> scene"""
    pcs, Rs, sc_, als = [], [], [], []
    corners = ((4.3, 4.3), (11.7, 4.3), (4.3, 11.7), (11.7, 11.7))
    gx = (W + 15) // 16
    for t, lst in enumerate(tiles):
        x0, y0 = 16 * (t % gx), 16 * (t // gx)
        for j, (a, centre, z) in enumerate(lst):
            px, py = (x0 + 8.0, y0 + 8.0) if centre else (x0 + corners[j % 4][0], y0 + corners[j % 4][1])
            sig = 2.2 if centre else 0.8
            pcs.append([px * z / F, py * z / F, z])
            sc_.append([sig * z / F, sig * 1.03 * z / F, 0.0])
            als.append(a)
    N = len(pcs)
    rng = np.random.default_rng(seed)
    return place(np.array(pcs), fronto(N), np.array(sc_), rng.normal(scale=0.3, size=(N, 3 * k)), np.array(als),
                 "identity", W, H, fx=F, cx=0.0, cy=0.0)


# ---------------------------------------------------------------- the median-tie stacks
TIE_LEN = 40
TIE_AT = (1, 31, 32, 33)   # list positions whose incoming tau is exactly 0.5 at the centre
FILL = 0.6                 # the fillers' alpha


def tie_stacks(k=1):
    """tie stacks, one per tile, 40 records each (depth order = list order), identity camera:
    - tie tiles: alpha 0.5 at position p - 1 and 0.25, 0.75 after it: the incoming tau is exactly 0.5
      at position p in TIE_AT (position 0 has nothing in front of it, its incoming tau is 1: the first
      tile puts the 0.5 there and the tie at 1).  The strict median is the record at p - 1; p = 32 puts
      the tie across the chunk boundary, p = 33 the median record itself in the second 32-record chunk;
    - stop tile: alpha 0.75 at 32 (incoming tau 1: the median, in the second chunk), 0.99 at 33 and
      34 (tau 2.5e-5: the walk stops after 34), then 0.5 at 35-39 that are never composited.  The
      median cannot be the record the walk stops at: alpha' <= 0.99 takes an incoming tau above 0.5 to
      no less than 0.005, so it is the last record of the chunk before the two that stop it;
    - clamp tile before: 0.5 at 30 (the median), alpha 1.0 at 31 (clamped to 0.99; incoming tau exactly
      0.5, so not the median), 0.5 at 32;
    - clamp tile median: 0.25 at 30, alpha 1.0 at 31 (incoming 0.75: the clamped record is the median).
    Everything else is a filler.  -> (scene, expected median_contrib at each tile's centre, tie[tiles])"""
    z = dyadic_depths(3.0, TIE_LEN)
    lists, medc, tie = [], [], []

    def tile(at):
        lists.append([(at[j], True, z[j]) if j in at else (FILL, False, z[j]) for j in range(TIE_LEN)])

    for p in TIE_AT:
        tile({p - 1: 0.5, p: 0.25, p + 1: 0.75})
        medc.append(p)
        tie.append(True)
    tile({32: 0.75, 33: 0.99, 34: 0.99, **{j: 0.5 for j in range(35, 40)}})
    medc.append(33)
    tie.append(False)
    tile({30: 0.5, 31: 1.0, 32: 0.5})
    medc.append(31)
    tie.append(True)
    tile({30: 0.25, 31: 1.0, 32: 0.5})
    medc.append(32)
    tie.append(False)
    sc = exact_stacks(lists, 16 * len(lists), 16, seed=21, k=k)
    return sc, np.array(medc), np.array(tie)


def centres(n):
    """(ys, xs) of the centre pixels of the first n tiles of a one-row frame"""
    return np.full(n, 8), 16 * np.arange(n) + 8


def tie_claims(sc, pre, bins, fwd, medc, tie):
    """the lists, the exact ties at the centres and the median record of each centre"""
    _, ranges, gsid, _ = bins
    n = len(medc)
    assert list(ranges[:, 1] - ranges[:, 0]) == [TIE_LEN] * n
    for t in range(n):   # draw order = list order
        assert list(gsid[ranges[t, 0]:ranges[t, 1]]) == list(range(TIE_LEN * t, TIE_LEN * (t + 1)))
    ys, xs = centres(n)
    assert np.array_equal(fwd["ties"][ys, xs], tie)
    assert np.array_equal(fwd["median_contrib"][ys, xs], medc)
    return ys, xs


def test_tie_stacks_reach_their_edges():
    sc, medc, tie = tie_stacks()
    pre, bins, _ = oracle_frame(sc)
    margins(sc, pre, bins)
    fwd = sg.render_geometry(sc["H"], sc["W"], pre, sc["alphas"], bins, exact=True)
    ys, xs = tie_claims(sc, pre, bins, fwd, medc, tie)
    # the model is exact at the centres: u on the pixel, alpha' = alpha, tau products of 1/2, 1/4, 3/4
    assert np.array_equal(pre["u"][medc - 1 + TIE_LEN * np.arange(len(medc))], np.stack([xs, ys], 1))
    # a tie at every position of TIE_AT, in order, and the median in the second chunk in two tiles
    assert np.array_equal(medc[:len(TIE_AT)], TIE_AT) and (medc - 1 >= 32).sum() >= 2
    # under `tau >= 0.5` the median of a tie tile would move one record on
    non_strict = np.where(tie, medc + 1, medc)
    assert not np.array_equal(non_strict, fwd["median_contrib"][ys, xs])
    # stop tile: terminated right after position 34, two records after its median
    t = len(TIE_AT)
    assert fwd["contrib"][8, 16 * t + 8] == 35 and fwd["final_tau"][8, 16 * t + 8] < so.TAU_STOP
    # clamp tiles: the record at 31 (alpha 1.0) is clamped at the centre
    for t in (t + 1, t + 2):
        e = so._eval(pre["M"][TIE_LEN * t + 31], pre["u"][TIE_LEN * t + 31], np.array([16.0 * t + 8]), np.array([8.0]))
        assert e["G"][0] == 0 and sc["alphas"][TIE_LEN * t + 31] * np.exp(-0.5 * e["G"][0]) > so.ALPHA_CLAMP
    # the median depth is the median record's hit depth: its own Z
    assert np.array_equal(fwd["median_depth"][ys, xs], pre["pc"][medc - 1 + TIE_LEN * np.arange(len(medc)), 2])


# ---------------------------------------------------------------- near and far
NF_Z = dyadic_depths(3.0, 6)
NF_NEAR, NF_FAR = float(NF_Z[2]), 3.25


def near_far_scene(k=1):
    """three exact stacks (identity camera) for near = NF_NEAR, far = NF_FAR, six records each with
    alphas 0.3-0.55 and depths 1/2048 apart:
    tile 0: hits at NF_Z, NF_NEAR - 2/2048 ... NF_NEAR + 3/2048, one exactly at near (position 2);
    tile 1: every hit between 2.5 and 2.51, below near (m = 0 for every record);
    tile 2: every hit beyond far (m > 1).  -> scene"""
    al = [0.3, 0.45, 0.55, 0.4, 0.5, 0.35]
    zs = (NF_Z, dyadic_depths(2.5, 6), dyadic_depths(3.5, 6))
    return exact_stacks([[(a, True, z) for a, z in zip(al, zz)] for zz in zs], 48, 16, seed=22, k=k)


def test_near_far_scene_reaches_its_edges():
    sc = near_far_scene()
    pre, bins, _ = oracle_frame(sc)
    margins(sc, pre, bins)
    fwd = sg.render_geometry(sc["H"], sc["W"], pre, sc["alphas"], bins, NF_NEAR, NF_FAR, exact=True)
    live = fwd["contrib"] > 0
    t0, t1, t2 = (live & (np.arange(48)[None, :] // 16 == t) for t in range(3))
    assert t0.sum() > 30 and t1.sum() > 30 and t2.sum() > 30
    # tile 0: hits exactly at near, composited before and after hits on both sides of it
    assert fwd["at_near"][t0].mean() > 0.9 and not fwd["at_near"][~t0].any()
    assert pre["pc"][2, 2] == NF_NEAR and (pre["pc"][:2, 2] < NF_NEAR).all() and (pre["pc"][3:6, 2] > NF_NEAR).all()
    assert (fwd["distortion"][t0] > 0).mean() > 0.5
    # tile 1: every hit below near: no distortion and no moments, exactly; the median is still there
    assert (pre["pc"][6:12, 2] < NF_NEAR).all()
    assert not fwd["distortion"][t1].any() and not fwd["moments"][:, t1].any()
    assert (fwd["median_depth"][t1] > 0).all()
    # tile 2: every hit beyond far: m > 1, so D > A
    assert (pre["pc"][12:, 2] > NF_FAR).all()
    assert (fwd["moments"][0][t2] > fwd["alpha"][t2]).all() and (fwd["distortion"][t2] > 0).mean() > 0.5
    assert not fwd["ambiguous"][live].mean() > 0.02


EXTREME = (1e-3, 1e4)


def extreme_scene(k=4):
    return random_scene(700, 160, 96, k, cam="posed_a", seed=23, spread=1.1, z=(1.0, 6.0))


def fp32_distortion(H, W, pre, alphas, bins, near, far):
    """distortion accumulated as the kernel does, w (m (m A - 2 D) + D2) with A, D, D2 its running sums,
    in fp32 with every operation rounded (no fma: an upper estimate of the kernel's rounding); w and m
    from fp64, rounded to fp32"""
    f = np.float32
    out = np.zeros((H, W), np.float32)
    _, ranges, gsid, _ = bins
    for t, X, Y in so._tiles(H, W, ranges):
        tau = np.ones(len(X))
        A, D, D2, dist = (np.zeros(len(X), np.float32) for _ in range(4))
        for i in gsid[ranges[t, 0]:ranges[t, 1]]:
            e = so._eval(pre["M"][i], pre["u"][i], X.astype(np.float64), Y.astype(np.float64))
            ap = np.minimum(so.ALPHA_CLAMP, float(alphas[i]) * np.exp(-0.5 * e["G"]))
            on = (tau >= so.TAU_STOP) & (ap >= so.ALPHA_SKIP)
            w = np.where(on, tau * ap, 0.0).astype(f)
            m = np.where(on, sg.m_of(e["z"], near, far), 0.0).astype(f)
            dist = dist + w * (m * (m * A - f(2) * D) + D2)
            A, D, D2 = A + w, D + w * m, D2 + (w * m) * m
            tau = np.where(on, tau * (1 - ap), tau)
        out[Y, X] = dist
    return out


def test_extreme_near_far_cancels_within_the_conditioning_bound():
    """near = 1e-3, far = 1e4: every m lies within 1e-3 of 1, so the moment form m^2 A + D2 - 2 m D of
    each record's term cancels terms of size A down to A (dm)^2.  The geometry planes are held to
    |distortion - model| <= 1e-4 cond + 2^-20 A^2 with cond = sum w (m^2 A + D2 + 2 m D) = 2 (A D2 + D^2),
    the pixel's conditioning: each record's term carries a few fp32 roundings of its three summands,
    about 2^-22 w (m^2 A + D2 + 2 m D), and their sum 2^-22 cond, 400 times below the bound.  A bound
    relative to the distortion itself cannot hold here: the fp32 error exceeds 1e-4 |distortion|."""
    sc = extreme_scene()
    pre, bins, _ = oracle_frame(sc)
    margins(sc, pre, bins)
    H, W = sc["H"], sc["W"]
    near, far = EXTREME
    fwd = sg.render_geometry(H, W, pre, sc["alphas"], bins, near, far)
    live = fwd["count"] > 1
    assert live.mean() > 0.3 and not fwd["ambiguous"][live].mean() > 0.02
    zs = pre["depths"][pre["keep"]]
    assert (1 - sg.m_of(zs, near, far) < 1.1e-3).all()
    A, D, D2 = fwd["alpha"], fwd["moments"][0], fwd["moments"][1]
    cond = 2 * (A * D2 + D * D)
    dist = fwd["distortion"]
    assert (dist[live] / cond[live]).max() < 1e-5
    got = fp32_distortion(H, W, pre, sc["alphas"], bins, near, far).astype(np.float64)
    err = np.abs(got - dist)
    assert (err[live] <= 1e-4 * cond[live] + 2.0 ** -20 * A[live] ** 2).all()
    assert (err[live] <= 2.0 ** -19 * cond[live] + 2.0 ** -20 * A[live] ** 2).all()   # far inside the bound
    assert (err[live] > 1e-4 * np.abs(dist[live])).any()


def coplanar_scene(k=1):
    """14 overlapping fronto-parallel disks at one exact depth (identity camera, 64 x 48 frame): every
    hit depth is that Z"""
    rng = np.random.default_rng(24)
    z = dyadic_depths(2.7, 1)[0]
    N = 14
    x, y = rng.uniform(10, 54, N), rng.uniform(10, 38, N)
    sig = rng.uniform(2.0, 6.0, N)
    sc = place(np.stack([x * z / F, y * z / F, np.full(N, z)], 1), fronto(N),
               np.stack([sig * z / F, sig * 1.1 * z / F, np.zeros(N)], 1), rng.normal(scale=0.3, size=(N, 3 * k)),
               rng.uniform(0.3, 0.7, N), "identity", 64, 48, fx=F, cx=0.0, cy=0.0)
    return sc, z


# ---------------------------------------------------------------- the model's claims on the edge scenes
def geometry_claims(fwd):
    """median_contrib 0 exactly where contrib is 0 and never beyond it; a pixel with one contributing
    record has distortion exactly 0 (its only term is w (m^2 0 + 0 - 2 m 0))"""
    con, medc = fwd["contrib"], fwd["median_contrib"]
    assert np.array_equal(medc == 0, con == 0)
    assert (medc <= con).all()
    one = fwd["count"] == 1
    assert not fwd["distortion"][one].any()
    assert (fwd["count"] <= con).all() and np.array_equal(fwd["count"] == 0, con == 0)
    return int(one.sum())


EDGE_SCENES = ["stack", "dense", "special_identity", "special_posed_b", "97x61", "17x9", "7x5"] + \
    ["random_%s_%d" % (c, k) for c in ("posed_a", "posed_b") for k in (1, 4, 9, 16)]


def edge_scene(name):
    """the scenes the geometry kernels are run on at the edges, by name: the surfel edge scenes, the
    odd frames of test_gpu_surfel_edges.test_odd_frames, random scenes with culled surfels at every SH
    degree and both posed cameras, and the tie and near/far stacks"""
    if name == "stack":
        return stack_scene()[0]
    if name == "dense":
        return dense_scene()
    if name.startswith("special_"):
        return special_scene(cam=name[len("special_"):])
    if name.startswith("random_"):
        cam, k3 = name[len("random_"):].rsplit("_", 1)
        return with_culled(random_scene(700, 160, 96, int(k3), cam=cam, seed=31 + int(k3), spread=1.1))
    if name == "tie":
        return tie_stacks()[0]
    if name == "near_far":
        return near_far_scene()
    W, H = (int(v) for v in name.split("x"))
    return random_scene(max(40, W * H // 20), W, H, 4, cam="posed_a", seed=W, spread=1.1)


def near_far_pairs(sc):
    """(near, far) cutting through the kept surfels' depths (far above them all), and (near, far) with far
    below the farthest of them"""
    z = pre_of(sc)["depths"]
    lo, hi = np.quantile(z[z > 0], [0.05, 0.95])
    return [(float(lo + 0.4 * (hi - lo)), 100.0), (0.2, float(lo + 0.5 * (hi - lo)))]


@pytest.mark.parametrize("pair", [0, 1])
@pytest.mark.parametrize("name", ["stack", "dense", "special_identity", "special_posed_b", "97x61", "17x9", "7x5",
                                  "random_posed_b_9", "tie", "near_far"])
def test_geometry_claims_on_the_edge_scenes(name, pair):
    """at the first (near, far) of near_far_pairs surfels lie on both sides of near; at the second a
    surfel beyond far composites (m > 1 there); and geometry_claims"""
    sc = edge_scene(name)
    near, far = near_far_pairs(sc)[pair]
    pre, bins, _ = oracle_frame(sc)
    H, W = sc["H"], sc["W"]
    fwd = sg.render_geometry(H, W, pre, sc["alphas"], bins, near, far)
    ones = geometry_claims(fwd)
    if name in ("97x61", "17x9", "tie"):   # pixels reached by one record only
        assert ones > 0
    if name == "stack":   # list positions 31-33 and the stop tiles: medians in the second chunk too
        assert (fwd["median_contrib"] > 32).any()
    z = pre["depths"]
    if pair == 0:
        assert (z[z > 0] < near).any() and (z > near).any()
    else:
        hit = sg.composited_at(H, W, pre, sc["alphas"], bins, fwd, np.ones((H, W), bool))
        assert (hit & (z > far)).any()


def test_geometry_claims_on_the_dead_tiles():
    """the 4K frame at 1 km, on its first three tile rows: the live hits lie beyond far = 100 (m > 1)
    and the dead tiles composite nothing"""
    sc, dead = dead_scene()
    pre = so.preprocess(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                        sc["fy"], sc["cx"], sc["cy"])
    bins = so.bin_f32(sc["H"], sc["W"], pre)
    dead_t = dead_claims(sc, dead, bins)
    gx = sc["W"] // 16
    r = bins[1].copy()
    r[3 * gx:] = 0
    fwd = sg.render_geometry(sc["H"], sc["W"], pre, sc["alphas"], (bins[0], r, bins[2], bins[3]), 0.2, 100.0)
    geometry_claims(fwd)
    band = np.zeros((sc["H"], sc["W"]), bool)
    band[:48] = True
    dpx = np.repeat(np.repeat(dead_t, 16, 0), 16, 1)
    assert not fwd["contrib"][dpx].any()
    live = band & (fwd["contrib"] > 0)
    assert live.sum() > 1000 and (fwd["moments"][0][live] > fwd["alpha"][live]).all()


def test_coplanar_disks_have_no_distortion():
    """every hit at one depth: every m equal, so each term w (m^2 A + D2 - 2 m D) is 0 up to fp64
    rounding, and the median depth is that depth exactly"""
    sc, z = coplanar_scene()
    pre, bins, _ = oracle_frame(sc)
    margins(sc, pre, bins)
    fwd = sg.render_geometry(48, 64, pre, sc["alphas"], bins, 0.2, 100.0)
    geometry_claims(fwd)
    A, D, D2 = fwd["alpha"], fwd["moments"][0], fwd["moments"][1]
    cond = 2 * (A * D2 + D * D)
    many = fwd["count"] > 2
    assert many.sum() > 200
    assert (np.abs(fwd["distortion"]) <= 1e-14 * cond).all()
    med = fwd["median_contrib"] > 0
    assert (fwd["median_depth"][med] == z).all() and med.sum() > 500
