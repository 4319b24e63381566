"""2D Gaussian Splatting edge scenes, checked without a GPU.

1. The fp64 oracle's backward (oracle/surfel_oracle.py) against central differences of its own
   forward at two posed cameras (generic rotations, twc off every axis, tcw = -Rcw twc), every
   parameter and the screen-space shift, SH degrees 0-3, with an edge-on, a clamped and a
   flipped-normal surfel.  At the identity camera Rcw and Rcw^T, pws - twc and pc, tcw and twc
   give the same numbers; here they do not.
2. The scene generators of tests/test_gpu_surfel_edges.py, each checked with the oracle alone to
   reach the edge it claims (list lengths, chunk edges, early termination, the clamp, both
   evaluation branches, cull extents of -inf and +inf, areas at the 2^24 cap, 64-bit depth keys),
   and to keep the margins under which binning the oracle on its own fp32 (u, depth, area) gives
   the kernels' tile lists: depth keys (millimetres) at least 0.01 from an integer, so surfels
   sharing a tile are either in one key (ordered by index on both sides) or more than 1e-5 apart
   relative, and fp64 binning half-extents at least 1e-3 from an integer (or at the cap).
"""
import numpy as np
import pytest

from oracle import surfel_oracle as so

f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)


# ---------------------------------------------------------------- cameras and surfel frames
def rot(axis, ang):
    """rotation matrix about a (normalised) axis"""
    k = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(ang) * Kx + (1 - np.cos(ang)) * Kx @ Kx


def quat(R):
    """unit quaternion (w, x, y, z) of a rotation matrix (Shepperd's branch choice)"""
    t = np.trace(R)
    cands = [1 + t, 1 + R[0, 0] - R[1, 1] - R[2, 2], 1 - R[0, 0] + R[1, 1] - R[2, 2], 1 - R[0, 0] - R[1, 1] + R[2, 2]]
    i = int(np.argmax(cands))
    s = np.sqrt(cands[i]) * 2
    if i == 0:
        q = [s / 4, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s]
    elif i == 1:
        q = [(R[2, 1] - R[1, 2]) / s, s / 4, (R[0, 1] + R[1, 0]) / s, (R[0, 2] + R[2, 0]) / s]
    elif i == 2:
        q = [(R[0, 2] - R[2, 0]) / s, (R[0, 1] + R[1, 0]) / s, s / 4, (R[1, 2] + R[2, 1]) / s]
    else:
        q = [(R[1, 0] - R[0, 1]) / s, (R[0, 2] + R[2, 0]) / s, (R[1, 2] + R[2, 1]) / s, s / 4]
    return np.array(q)


CAMERAS = {
    "identity": (np.eye(3), np.zeros(3)),
    # generic rotations (not about one axis) and camera centres off every axis
    "posed_a": (rot([0.3, -0.5, 0.8], 0.41), np.array([0.31, -0.22, 0.17])),
    "posed_b": (rot([-0.7, 0.2, 0.45], -0.83), np.array([-0.45, 0.38, -0.29])),
}


def camera(name):
    """-> (Rcw, tcw, twc) in fp64 with tcw = -Rcw twc"""
    Rcw, twc = CAMERAS[name]
    return Rcw, -Rcw @ twc, twc


def place(pc, Rc, scales, shs, alphas, cam, W, H, fx=None, fy=None, cx=None, cy=None):
    """surfels given in the camera frame (centres pc, rotations Rc whose columns are the camera-frame
    R e0, R e1, R e2) -> a scene dict in world coordinates for `cam`, fp32"""
    Rcw, tcw, twc = camera(cam)
    pws = (np.asarray(pc, np.float64) - tcw) @ Rcw
    rots = np.stack([quat(Rcw.T @ R) for R in Rc]) if len(Rc) else np.zeros((0, 4))
    fx = 0.8 * W if fx is None else fx
    return dict(pws=f32(pws), rots=f32(rots), scales=f32(scales), shs=f32(shs), alphas=f32(alphas), Rcw=f32(Rcw),
                tcw=f32(tcw), twc=f32(twc), fx=float(fx), fy=float(fx if fy is None else fy),
                cx=float(W / 2 - 0.3 if cx is None else cx), cy=float(H / 2 + 0.2 if cy is None else cy), W=W, H=H)


def random_rotations(rng, N):
    q = rng.normal(size=(N, 4))
    q /= np.linalg.norm(q, axis=1)[:, None]
    return so.quat_R(q)


def pre_of(sc):
    return so.preprocess(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                         sc["fy"], sc["cx"], sc["cy"])


def ext_margin_bad(pre):
    """kept surfels whose fp64 binning half-extent lies within 1e-3 of an integer (below the cap)"""
    e = pre["ext"]
    return pre["keep"] & ((np.abs(e - np.round(e)) < 1e-3) & (e < so.AREA_CAP - 1)).any(axis=1)


def with_margins(sc, rng, tries=20):
    """nudges the scales of surfels without the half-extent margin until every one has it"""
    for _ in range(tries):
        bad = ext_margin_bad(pre_of(sc))
        if not bad.any():
            return sc
        sc["scales"][bad, :2] = f32(sc["scales"][bad, :2] * rng.uniform(1.001, 1.01, (bad.sum(), 1)))
    raise AssertionError("could not give every surfel its half-extent margin")


def mm_depths(rng, N, lo, hi):
    """camera depths at the middle of a millimetre: the depth key floor(1000 z) has a 0.5 margin"""
    return (rng.integers(int(lo * 1000), int(hi * 1000), N) + 0.5) / 1000.0


def random_scene(N, W, H, k, cam="identity", seed=0, z=(2.0, 6.0), spread=1.0, size=(0.02, 0.15),
                 alpha=(0.05, 0.95)):
    """test_gpu_surfel.scene at any camera: random disks over the frame, depths on the millimetre
    lattice, binning half-extents off the integers"""
    rng = np.random.default_rng(seed)
    fx = 0.8 * W
    zz = mm_depths(rng, N, *z)
    pc = np.stack([rng.uniform(-spread, spread, N) * zz * W / (2 * fx),
                   rng.uniform(-spread, spread, N) * zz * H / (2 * fx), zz], 1)
    scales = np.stack([rng.uniform(*size, N), rng.uniform(*size, N), rng.uniform(0.0, 0.05, N)], 1)
    sc = place(pc, random_rotations(rng, N), scales, rng.normal(scale=0.3, size=(N, 3 * k)),
               rng.uniform(*alpha, N), cam, W, H)
    return with_margins(sc, rng)


def edge_on(c):
    """camera-frame rotation of a disk at c seen edge-on: its normal 0.02 rad off perpendicular to
    the view ray, so the side it faces (the normal's flip) is not decided by rounding"""
    v = np.asarray(c, np.float64) / np.linalg.norm(c)
    n = np.cross(v, [0.0, 1.0, 0.0])
    n = n / np.linalg.norm(n) + 0.02 * v
    n /= np.linalg.norm(n)
    e1 = np.array([0.0, 1.0, 0.0]) - n[1] * n
    e1 /= np.linalg.norm(e1)
    return np.stack([np.cross(e1, n), e1, n], 1)


def fronto(N):
    """camera-frame rotations of disks facing the camera (R e2 = -z)"""
    return np.repeat(np.diag([1.0, -1.0, -1.0])[None], N, axis=0)


# ---------------------------------------------------------------- edge scenes
STACK_LENS = (31, 32, 33, 64, 65, 96, 97)
STOP_AT = (31, 32, 33)   # list positions of the last composited record at the stop tiles' centres
CLAMP_ALPHAS = (0.99, float(np.nextafter(np.float32(0.99), np.float32(1.0))), 1.0, 0.99)  # positions 30-33
TILE_Z = 3.0


def stack_scene(k=1):
    """one stack of concentric fronto-parallel disks per tile, centred 0.2 px from the pixel (8, 8) of the tile,
    sigma 2.2 px (binning half-extent 7: one tile each), identity camera.  Tiles in order:
    - lists of every length in STACK_LENS with alpha 0.05 (every record composited at the centre);
    - stop tiles: alpha 0.1, then two of alpha 1.0 at positions m - 1, m (m in STOP_AT), 40 long:
      the centre pixel terminates after position m;
    - a tiny-alpha tile: alphas 0.001 (cull -inf) and 0.002 alternating, 8 long;
    - a clamp tile: alpha 0.05, CLAMP_ALPHAS at positions 30-33, 40 long, in the partial last tile
      column of the odd frame width (16 * tiles + 13) and height 21.
    -> (scene, expected list length per tile)"""
    lists = []
    for L in STACK_LENS:
        lists.append(np.full(L, 0.05))
    for m in STOP_AT:
        a = np.full(40, 0.1)
        a[m - 1:m + 1] = 1.0
        lists.append(a)
    lists.append(np.tile([0.001, 0.002], 4))
    a = np.full(40, 0.05)
    a[30:34] = CLAMP_ALPHAS
    lists.append(a)
    W, H = 16 * (len(lists) - 1) + 13, 21
    f, cx, cy = 40.0, 0.0, 0.0
    pcs, alphas = [], []
    for t, al in enumerate(lists):
        # 0.2 px right of the pixel (8, 8): alpha 1.0 clamps there (G ~ 0.008) while G3 and G2 differ
        # by more than the oracle's ambiguity margin
        x = (16 * t + 8 if t < len(lists) - 1 else W - 3) + 0.2   # the last stack inside the partial tile
        for j in range(len(al)):
            z = TILE_Z + 0.001 * j + 0.0005   # one millimetre key per position: draw order = list order
            pcs.append([(x - cx) * z / f, (8 - cy) * z / f, z])
        alphas.append(al)
    pc, alphas = np.array(pcs), np.concatenate(alphas)
    N = len(pc)
    s = 2.2 * TILE_Z / f
    rng = np.random.default_rng(3)
    sc = place(pc, fronto(N), np.stack([np.full(N, s), np.full(N, s * 1.03), np.zeros(N)], 1),
               rng.normal(scale=0.3, size=(N, 3 * k)), alphas, "identity", W, H, fx=f, cx=cx, cy=cy)
    return sc, [len(a) for a in lists]


def dense_scene(k=4, seed=5):
    """3000 large, mostly opaque surfels over a 64 x 48 frame at posed camera A: lists of hundreds
    of records, most pixels terminate early"""
    return random_scene(3000, 64, 48, k, cam="posed_a", seed=seed, size=(0.1, 0.4), alpha=(0.4, 0.95))


def special_scene(k=4, cam="posed_b"):
    """one surfel per kind, in the camera frame of `cam`, 96 x 64 frame:
    0 edge-on (normal across the view ray)      1 grazing (normal 85 deg off the ray)
    2 sub-pixel (drawn by the filter only)       3 needle (100:1)
    4 frame-sized                                5 off-screen centre, footprint reaching in
    6 t-level ellipse unbounded (cull +inf)      7 alpha 0.0015 (cull -inf)
    8 binning half-extent at the 2^24 cap: a large disk whose near edge grazes the camera plane
    9 fronto-parallel, normal flipped (R e2 facing away from the camera)"""
    W, H = 96, 64
    f = 0.8 * W
    cx, cy = W / 2 - 0.3, H / 2 + 0.2
    px = lambda x, y, z: [(x - cx) * z / f, (y - cy) * z / f, z]
    Rc, pc, sz, al = [], [], [], []

    def add(R, c, s, a):
        Rc.append(R); pc.append(c); sz.append(s); al.append(a)

    c0 = px(30.3, 20.6, 3.0005)
    add(edge_on(c0), c0, (0.3, 0.2), 0.8)
    c1 = px(60.2, 40.7, 4.0005)
    add(rot([1.0, 0.0, 0.0], np.deg2rad(85)) @ np.diag([1.0, -1.0, -1.0]), c1, (0.4, 0.3), 0.7)
    add(fronto(1)[0], px(12.4, 50.3, 5.0005), (0.004, 0.004), 0.9)
    add(rot([0.0, 0.0, 1.0], 0.3) @ fronto(1)[0], px(70.1, 15.2, 3.5005), (1.2, 0.012), 0.75)
    add(rot([0.2, 0.1, 1.0], 0.5) @ fronto(1)[0], px(47.6, 31.9, 6.0005), (8.0, 6.0), 0.1)
    add(fronto(1)[0], px(-9.7, 30.4, 2.5005), (0.5, 0.4), 0.6)
    # m3 = (tu.z, tv.z, pc.z) with tu.z^2 + tv.z^2 = pc.z^2 / 10: bounded at level 9, not at t > 10
    z6 = 5.0005
    tilt = np.arcsin(z6 / np.sqrt(10) / 2.0)
    add(rot([1.0, 0.0, 0.0], -tilt) @ fronto(1)[0], px(20.2, 12.3, z6), (0.1, 2.0), 0.8)
    add(fronto(1)[0], px(80.3, 50.6, 4.5005), (0.3, 0.3), 0.0015)
    # the 3-sigma disk's nearest point 4 um in front of the camera plane: D / pc.z^2 ~ 4e-6, its
    # sign safe in fp32, the half-extent over 2^24 px
    z8 = 2.0005
    tilt8 = np.arcsin((z8 - 4e-6) / 3.0 / 1.5)
    add(rot([1.0, 0.0, 0.0], -tilt8) @ fronto(1)[0], px(50.4, 40.2, z8), (30.0, 1.5), 0.3)
    add(np.diag([1.0, 1.0, 1.0]), px(40.3, 50.2, 2.2005), (0.2, 0.15), 0.6)
    N = len(pc)
    rng = np.random.default_rng(8)
    scales = np.concatenate([np.array(sz), np.zeros((N, 1))], 1)
    return place(np.array(pc), Rc, scales, rng.normal(scale=0.3, size=(N, 3 * k)), al, cam, W, H, fx=f, cx=cx, cy=cy)


DEAD_W, DEAD_H = 3840, 2160


def dead_scene(k=1, seed=11):
    """3840 x 2160 at about 1 km: one to three fronto-parallel disks inside each tile (binning
    half-extent <= 7 around a centre in the tile's middle), checkerboard tiles of alpha 0.0015 that
    composite nothing.  Depth keys reach 2^20 and the tile index 15 bits: 64-bit keys."""
    rng = np.random.default_rng(seed)
    gx, gy = DEAD_W // 16, DEAD_H // 16
    f = 0.8 * DEAD_W
    cx, cy = DEAD_W / 2, DEAD_H / 2
    cnt = rng.integers(1, 4, gx * gy)
    tile = np.repeat(np.arange(gx * gy), cnt)
    N = len(tile)
    tx, ty = tile % gx, tile // gx
    x = 16 * tx + 8 + rng.integers(-1, 2, N) + 0.25
    y = 16 * ty + 8 + rng.integers(-1, 2, N) + 0.25
    z = 1000.0 + 0.0005 + 0.02 * rng.integers(0, 1000, N)   # keys ~1e6, 2e-5 apart relative, margin 0.5
    pc = np.stack([(x - cx) * z / f, (y - cy) * z / f, z], 1)
    dead = ((tx + ty) % 2) == 1
    alphas = np.where(dead, 0.0015, rng.uniform(0.3, 0.9, N))
    s = rng.uniform(0.9, 1.5, N) * z / f   # sigma 0.9-1.5 px
    sc = place(pc, fronto(N), np.stack([s, s * 1.1, np.zeros(N)], 1), rng.normal(scale=0.3, size=(N, 3 * k)),
               alphas, "identity", DEAD_W, DEAD_H, fx=f, cx=cx, cy=cy)
    return with_margins(sc, rng), dead


# ---------------------------------------------------------------- oracle claims
def margins(sc, pre, bins):
    """the margins of an exact independent binning: depth keys at least 0.01 from an integer, surfels
    sharing a tile either in one key or more than 1e-5 apart relative, fp64 binning half-extents at
    least 1e-3 from an integer (or at the cap)"""
    k = pre["keep"]
    key = pre["depths"][k] * 1000
    fr = key - np.floor(key)
    assert fr.min() >= 0.01 and fr.max() <= 0.99, (fr.min(), fr.max())
    assert not ext_margin_bad(pre).any()
    _, ranges, gsid, _ = bins
    d = pre["depths"]
    for r0, r1 in ranges:
        if r1 - r0 < 2:
            continue
        dz = np.sort(d[gsid[r0:r1]])
        gap = np.diff(dz)
        same = np.floor(dz[1:] * 1000) == np.floor(dz[:-1] * 1000)
        assert (same | (gap > 1e-5 * dz[1:])).all()


def composited_pairs(sc, pre, bins, fwd):
    """the branch (G3 <= G2) of every composited (pixel, surfel) pair, and whether any pixel had its
    alpha' clamped: -> (branches, clamped)"""
    H, W = sc["H"], sc["W"]
    _, ranges, gsid, _ = bins
    alphas = np.asarray(sc["alphas"], np.float64)
    b3s, clamped = [], False
    for t, X, Y in so._tiles(H, W, ranges):
        tau = np.ones(len(X))
        for j, i in enumerate(gsid[ranges[t, 0]:ranges[t, 1]]):
            e = so._eval(pre["M"][i], pre["u"][i], X.astype(np.float64), Y.astype(np.float64))
            ag = alphas[i] * np.exp(-0.5 * e["G"])
            on = (tau >= so.TAU_STOP) & (np.minimum(so.ALPHA_CLAMP, ag) >= so.ALPHA_SKIP)
            b3s.append(e["b3"][on])
            clamped |= bool((on & (ag > so.ALPHA_CLAMP)).any())
            tau = np.where(on, tau * (1 - np.minimum(so.ALPHA_CLAMP, ag)), tau)
    return np.concatenate(b3s) if b3s else np.zeros(0, bool), clamped


def oracle_frame(sc):
    pre = pre_of(sc)
    bins = so.bin_f32(sc["H"], sc["W"], pre)
    fwd = so.render(sc["H"], sc["W"], pre, sc["alphas"], bins)
    return pre, bins, fwd


def stack_claims(sc, lens, pre, bins, fwd):
    _, ranges, _, _ = bins
    got = ranges[:, 1] - ranges[:, 0]
    assert list(got[:len(lens)]) == lens, got
    con, tau = fwd["contrib"], fwd["final_tau"]
    n = len(STACK_LENS)
    for t, L in enumerate(STACK_LENS):   # every record composited at the centre pixel
        assert con[8, 16 * t + 8] == L
    for t, m in enumerate(STOP_AT):      # terminated right after position m
        c = con[8, 16 * (n + t) + 8]
        assert c == m + 1 and tau[8, 16 * (n + t) + 8] < so.TAU_STOP, (m, c)
    assert con[8, sc["W"] - 3] >= 32   # the clamp tile (the partial last one) reaches positions 30-33
    assert (fwd["contrib"][:, -6:] > 0).any()   # content in the partial tile column
    assert sc["W"] % 2 == 1


def dense_claims(bins, fwd):
    _, ranges, _, _ = bins
    lens = ranges[:, 1] - ranges[:, 0]
    assert lens.max() > 300 and (fwd["final_tau"] < so.TAU_STOP).mean() > 0.5
    assert fwd["contrib"].max() < lens.max()


def special_claims(sc, pre, bins, fwd, cull):
    """cull: the cull half-extents [N,2] (the oracle's at level t, or the kernels' records)"""
    assert pre["keep"].all()
    assert np.isposinf(cull[[6, 8]]).all() and np.isneginf(cull[7]).all()
    assert np.isfinite(cull[[0, 1, 2, 3, 4, 5, 9]]).all()
    assert (pre["areas"][8] == so.AREA_CAP).any() and (pre["ext"][8] >= so.AREA_CAP).any()
    assert (pre["areas"][[0, 1, 2, 3, 4, 5, 6, 7, 9]] < 2000).all()
    assert pre["sgn"][9] == -1 and (pre["sgn"][[2, 3]] == 1).all()
    b3, clamped = composited_pairs(sc, pre, bins, fwd)
    assert b3.any() and (~b3).any()
    for i in (0, 2, 4, 5, 8):   # each of these composites somewhere
        assert (fwd["contrib"] > 0).any()
    assert not fwd["ambiguous"].all()


def dead_claims(sc, dead, bins, fwd_contrib=None):
    """1-3 patches per tile, the dead checkerboard, 64-bit keys -> dead tiles [gy, gx]"""
    gx, gy = DEAD_W // 16, DEAD_H // 16
    _, ranges, _, keys = bins
    lens = ranges[:, 1] - ranges[:, 0]
    assert lens.min() >= 1 and lens.max() <= 3
    depth_bits = int((keys & 0xFFFFFFFF).max()).bit_length()
    tile_bits = (gx * gy - 1).bit_length()
    assert depth_bits >= 20 and tile_bits == 15 and depth_bits + tile_bits > 32
    per_tile = np.zeros(gx * gy, bool)
    tid = np.repeat(np.arange(gx * gy), lens)
    per_tile[tid] = dead[bins[2]]
    live = np.zeros(gx * gy, bool)
    np.logical_or.at(live, tid, ~dead[bins[2]])
    tiles_dead = ~live
    assert np.array_equal(tiles_dead.reshape(gy, gx), (np.add.outer(np.arange(gy), np.arange(gx)) % 2) == 1)
    return tiles_dead.reshape(gy, gx)


def cull_box(pre, alphas, dt=0.0):
    """the fp64 cull half-extents of the records: the footprint at level t = 2 ln(alpha / 0.002) + dt,
    -inf for alpha < 0.002, +inf where the t-level ellipse is unbounded"""
    a = np.asarray(alphas, np.float64)
    out = np.full((len(a), 2), -np.inf)
    ok = a >= np.float32(0.002)
    t = 2 * np.log(np.where(ok, a, 1.0) / 0.002) + dt
    for i in np.flatnonzero(ok):
        e, b = so.footprint(pre["M"][i:i + 1], pre["u"][i:i + 1], t[i])
        out[i] = e[0] if b[0] else np.inf
    return out


# ---------------------------------------------------------------- 1. oracle backward at posed cameras
H, W = 20, 36
FX = FY = 30.0
CX, CY = 17.3, 9.6


def fd_scene(k, cam, seed):
    """six surfels in front of `cam`: 0 edge-on, 1 clamped near its centre, 2 normal flipped, the
    rest random"""
    rng = np.random.default_rng(seed)
    N = 6
    pc = np.stack([rng.uniform(-0.8, 0.8, N), rng.uniform(-0.4, 0.4, N), rng.uniform(2.5, 4.0, N)], 1)
    Rc = list(random_rotations(rng, N))
    pc[0] = [0.1, 0.05, 3.0]
    Rc[0] = edge_on(pc[0])
    pc[1] = [-0.3, 0.1, 3.2]
    Rc[1] = rot([0.4, 0.3, 0.2], 0.3) @ fronto(1)[0]
    Rc[2] = rot([0.3, -0.2, 0.1], 0.4) @ np.eye(3)   # R e2 ~ +z: facing away, flipped
    scales = np.stack([rng.uniform(0.15, 0.4, N), rng.uniform(0.15, 0.4, N), rng.uniform(0.0, 0.1, N)], 1)
    scales[1, :2] = [0.7, 0.65]   # sigma over 5 px: alpha' above 0.99 at the pixels next to its centre
    alphas = rng.uniform(0.3, 0.9, N)
    alphas[1] = 0.9985
    Rcw, tcw, twc = camera(cam)
    pws = (pc - tcw) @ Rcw
    rots = np.stack([quat(Rcw.T @ R) for R in Rc])
    return dict(pws=pws, rots=rots, scales=scales, shs=rng.normal(scale=0.4, size=(N, 3 * k)), alphas=alphas,
                Rcw=Rcw, tcw=tcw, twc=twc)


def fd_loss(sc, bins, dl, delta=None):
    pre = so.preprocess(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], FX, FY, CX, CY)
    out = so.render(H, W, pre, sc["alphas"], bins, delta=delta)
    return (np.sum(out["image"] * dl[0]) + np.sum(out["depth"] * dl[1]) + np.sum(out["alpha"] * dl[2]) +
            np.sum(out["normal"] * dl[3]))


@pytest.mark.parametrize("cam", ["posed_a", "posed_b"])
@pytest.mark.parametrize("k", [1, 4, 9, 16])
def test_oracle_backward_at_posed_cameras(k, cam):
    sc = fd_scene(k, cam, seed=10 * k + len(cam))
    rng = np.random.default_rng(k + 7)
    dl = (rng.normal(size=(3, H, W)), rng.normal(size=(H, W)), rng.normal(size=(H, W)), rng.normal(size=(3, H, W)))
    pre = so.preprocess(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], FX, FY, CX, CY)
    assert pre["keep"].all()
    assert pre["sgn"][2] == -1 and pre["sgn"][1] == 1
    # the camera is posed: Rcw is not symmetric and twc, tcw differ
    assert np.abs(sc["Rcw"] - sc["Rcw"].T).max() > 0.1 and np.abs(sc["tcw"] - sc["twc"]).min() > 0.05
    bins = so.bin_f32(H, W, pre)
    fwd = so.render(H, W, pre, sc["alphas"], bins)
    assert not fwd["ambiguous"].any()
    assert (fwd["alpha"] > 0).mean() > 0.3
    e0 = so._eval(pre["M"][0], pre["u"][0], pre["u"][0][0] + np.array([1.5, -2.0]), pre["u"][0][1] + np.array([0.7, 1.0]))
    assert not e0["b3"].any()   # edge-on: the filter wins
    c = so._eval(pre["M"][1], pre["u"][1], np.round(pre["u"][1][:1]), np.round(pre["u"][1][1:]))
    assert sc["alphas"][1] * np.exp(-0.5 * c["G"][0]) > so.ALPHA_CLAMP
    g = so.preprocess_backward(pre, so.render_backward(H, W, pre, sc["alphas"], bins, fwd, *dl))
    eps = 1e-6
    for name, cols in (("pws", None), ("shs", None), ("alphas", None), ("scales", [0, 1]), ("rots", None)):
        arr = sc[name]
        fd = np.zeros_like(arr)
        for idx in np.ndindex(arr.shape):
            if cols is not None and idx[1] not in cols:
                continue
            keep = arr[idx]
            arr[idx] = keep + eps
            lp = fd_loss(sc, bins, dl)
            arr[idx] = keep - eps
            lm = fd_loss(sc, bins, dl)
            arr[idx] = keep
            fd[idx] = (lp - lm) / (2 * eps)
        an = g[name].reshape(arr.shape)
        if cols is not None:
            an, fd = an[:, cols], fd[:, cols]
        scale = np.abs(fd).max()
        assert scale > 0, name
        np.testing.assert_allclose(an, fd, atol=2e-5 * scale + 1e-7, err_msg=name)
    fd = np.zeros((6, 2))
    for i in range(6):
        for c_ in range(2):
            d = np.zeros((6, 2))
            d[i, c_] = eps
            fd[i, c_] = (fd_loss(sc, bins, dl, d) - fd_loss(sc, bins, dl, -d)) / (2 * eps)
    np.testing.assert_allclose(g["us"], fd, atol=2e-5 * np.abs(fd).max(), err_msg="delta")


def test_abs_rows_bound_the_rows():
    """render_backward(abs_rows=True) returns the same rows and, per entry, a sum of magnitudes at
    least as large as the entry"""
    sc = random_scene(40, 48, 32, 4, cam="posed_a", seed=3)
    pre, bins, fwd = oracle_frame(sc)
    rng = np.random.default_rng(1)
    dl = [rng.normal(size=s) for s in ((3, 32, 48), (32, 48), (32, 48), (3, 32, 48))]
    rows = so.render_backward(32, 48, pre, sc["alphas"], bins, fwd, *dl)
    rows2, ab = so.render_backward(32, 48, pre, sc["alphas"], bins, fwd, *dl, abs_rows=True)
    assert np.array_equal(rows, rows2)
    assert (ab >= np.abs(rows) * (1 - 1e-12)).all() and ab.max() > 0


# ---------------------------------------------------------------- 2. the generators reach their edges
def test_stack_scene_reaches_its_edges():
    sc, lens = stack_scene()
    pre, bins, fwd = oracle_frame(sc)
    margins(sc, pre, bins)
    stack_claims(sc, lens, pre, bins, fwd)
    _, clamped = composited_pairs(sc, pre, bins, fwd)
    assert clamped
    cull = cull_box(pre, sc["alphas"])
    assert np.isneginf(cull[sc["alphas"] < 0.002]).all()


def test_dense_scene_reaches_its_edges():
    sc = dense_scene()
    pre, bins, fwd = oracle_frame(sc)
    margins(sc, pre, bins)
    dense_claims(bins, fwd)


@pytest.mark.parametrize("cam", ["identity", "posed_b"])
def test_special_scene_reaches_its_edges(cam):
    sc = special_scene(cam=cam)
    pre, bins, fwd = oracle_frame(sc)
    margins(sc, pre, bins)
    special_claims(sc, pre, bins, fwd, cull_box(pre, sc["alphas"]))
    # the capped surfel covers the whole frame in the direction it is capped
    _, ranges, gsid, _ = bins
    assert (gsid == 8).sum() >= 0.5 * len(ranges)


def test_dead_scene_reaches_its_edges():
    sc, dead = dead_scene()
    pre = pre_of(sc)
    bins = so.bin_f32(sc["H"], sc["W"], pre)
    margins(sc, pre, bins)
    dead_claims(sc, dead, bins)


@pytest.mark.parametrize("W,H", [(97, 61), (17, 9), (7, 5)])
def test_odd_frames_have_content_in_the_last_column(W, H):
    sc = random_scene(max(40, W * H // 20), W, H, 1, cam="posed_a", seed=W, spread=1.1)
    pre, bins, fwd = oracle_frame(sc)
    margins(sc, pre, bins)
    assert W % 2 == 1 and (fwd["contrib"][:, -1] > 0).any()


@pytest.mark.parametrize("cam", list(CAMERAS))
def test_random_scenes_keep_their_margins(cam):
    for N in (1, 127, 128, 129, 2001):
        sc = random_scene(N, 160, 96, 4, cam=cam, seed=N)
        pre = pre_of(sc)
        margins(sc, pre, so.bin_f32(160, 96, pre))
