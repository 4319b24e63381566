"""The batch's tall frame (DESIGN 3.21) on the host: a numpy mirror of binning.cu's `key_plan`, checked
against the plan shapes test_gpu_binning's scenes reach, and the scene builders of
test_gpu_batch_edges.py checked to reach the tall-frame plan, row limit and capacity layout each is
built for.  A builder that misses its target fails here, not silently on the GPU.

The tall frame of C cameras of gx x gy tiles is gx x C gy tiles; its key plan is the single frame's at
height C gy 16, with the largest depth key over all C cameras.  Camera c's keys in it are its own single
frame's keys with c gx gy added to the tile field."""
import numpy as np
import pytest

from oracle import oracle as orc

from test_gpu_binning import PLANS, Scene, depth_for_key, key_plan_scene, widths


# ---------------------------------------------------------------- the key plan
def key_plan(H, W, dkmax):
    """binning.cu key_plan: -> dict(narrow, tbits, dbits, bits (digit width), shifts (one per pass),
    depth_bits (the depth-key bits the passes order))"""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    tbits = (gx * gy - 1).bit_length()
    dbits = 32 if dkmax == 0xFFFFFFFF else int(dkmax).bit_length()
    narrow = dbits < 32 and tbits + dbits <= 32
    if narrow:
        end = tbits + dbits
        bits = 9 if end > 0 and (end + 8) // 9 < (end + 7) // 8 else 8
        shifts = list(range(0, end, bits))
        depth_bits = dbits
    else:
        bits = 8
        shifts = list(range(0, dbits, 8)) + [32 + s for s in range(0, tbits, 8)]
        depth_bits = (dbits + 7) // 8 * 8
    return dict(narrow=narrow, tbits=tbits, dbits=dbits, bits=bits, shifts=shifts, depth_bits=depth_bits)


def tall_height(C, H):
    """kernels.h batch_height: C frames padded to whole tile rows"""
    return C * ((H + 15) // 16) * 16


def plan_shape(p):
    """(layout, passes, digit bits) of a plan"""
    return ("narrow" if p["narrow"] else "64bit", len(p["shifts"]), p["bits"])


# (tile bits, depth bits) of test_gpu_binning.PLANS -> the shape its docstring says each reaches:
# 1 to 4 passes of 8- or 9-bit digits, 32 and 33 bits, 32-bit and saturated depth keys in the 64-bit layout
SINGLE_PLAN_SHAPES = {
    (0, 8): ("narrow", 1, 8), (1, 8): ("narrow", 1, 9), (4, 12): ("narrow", 2, 8), (5, 12): ("narrow", 2, 9),
    (8, 16): ("narrow", 3, 8), (9, 16): ("narrow", 3, 9), (10, 17): ("narrow", 3, 9), (11, 17): ("narrow", 4, 8),
    (12, 20): ("narrow", 4, 8), (12, 21): ("64bit", 5, 8), (4, 32): ("64bit", 5, 8), (4, "saturated"): ("64bit", 5, 8),
}


@pytest.mark.parametrize("tbits,dbits", PLANS)
def test_key_plan_mirror_on_the_single_frame_plans(tbits, dbits):
    seed = tbits * 100 + (dbits if dbits != "saturated" else 99)
    H, W, T, (us, depths, areas) = key_plan_scene(tbits, dbits, seed=seed)
    P, ranges, gsid, keys = orc.bin(H, W, us, depths.copy(), areas.copy())
    p = key_plan(H, W, int((keys & np.uint64(0xFFFFFFFF)).max()))
    assert plan_shape(p) == SINGLE_PLAN_SHAPES[(tbits, dbits)]
    assert p["tbits"] == tbits and (dbits == "saturated" or p["dbits"] == dbits)
    # a narrow plan's passes cover exactly the tile and depth fields; a 64-bit one whole digits of each
    if p["narrow"]:
        assert p["shifts"][-1] < tbits + p["dbits"] <= len(p["shifts"]) * p["bits"]
    else:
        assert p["depth_bits"] >= p["dbits"] and p["shifts"][-1] >= 32


def test_key_plan_mirror_at_the_tall_frame():
    """the tall frame's plan from its height alone: C frames of one tile each sort like a C-tile column"""
    for C, H, W, dk, shape in ((2, 16, 16, 255, ("narrow", 1, 9)), (3, 16, 16, 65535, ("narrow", 2, 9)),
                               (8, 64, 64, 2 ** 25 - 1, ("narrow", 4, 8)), (8, 64, 64, 2 ** 26 - 1, ("64bit", 5, 8)),
                               (64, 16, 16, 2 ** 26 - 1, ("narrow", 4, 8)), (64, 16, 16, 2 ** 27 - 1, ("64bit", 5, 8))):
        assert plan_shape(key_plan(tall_height(C, H), W, dk)) == shape, (C, H, W, dk)
        assert plan_shape(key_plan(H, W, dk))[0] == "narrow"  # every single frame of these sorts 32-bit keys
    # config 5 of the benchmark: 8 cameras at 1920x1080 are 120 x 544 tiles, 16 tile bits; its scene's
    # depths (2 to 12 m from ring cameras 0.6 m off) have depth keys of 14 bits: four 8-bit passes.
    # Depth keys past 16 bits (65.5 m) would take it to the 64-bit layout.
    assert key_plan(tall_height(8, 1080), 1920, 12999)["tbits"] == 16
    assert plan_shape(key_plan(tall_height(8, 1080), 1920, 12999)) == ("narrow", 4, 8)
    assert plan_shape(key_plan(tall_height(8, 1080), 1920, 65536)) == ("64bit", 5, 8)
    # the row limit: 3 x 21845 and 64 x 1023 tile rows
    assert key_plan(tall_height(3, 16 * 21845), 16, 1)["tbits"] == 16
    assert key_plan(tall_height(64, 16 * 1023 - 5), 16, 1)["tbits"] == 16


# ---------------------------------------------------------------- batch scenes
def pad_cameras(cams):
    """per-camera (us, depths, areas) of different lengths -> [C, N, ...] arrays, every camera padded to
    the longest with rows culled by depth (-1: never binned, never culled in place)"""
    N = max(len(d) for _, d, _ in cams)
    C = len(cams)
    us = np.zeros((C, N, 2), np.float32)
    depths = np.full((C, N), -1.0, np.float32)
    areas = np.zeros((C, N, 2), np.int32)
    for c, (u, d, a) in enumerate(cams):
        us[c, :len(d)], depths[c, :len(d)], areas[c, :len(d)] = u, d, a
    return us, depths, areas


# name -> (C, the single frame's tile bits, depth-key bits per camera, what the tall frame reaches:
# (tall tile bits, tall depth bits, layout, passes, digit bits)).  "far": key_plan_scene at 14 depth
# bits everywhere, plus one Gaussian of a 22-bit depth key seen by camera 2 only.
BATCH_PLANS = {
    "tall_9": (2, 0, 8, (1, 8, "narrow", 1, 9)),
    "tall_17": (2, 0, 16, (1, 16, "narrow", 2, 9)),
    "tall_18": (3, 0, 16, (2, 16, "narrow", 2, 9)),
    "tall_25": (4, 1, 22, (3, 22, "narrow", 3, 9)),
    "tall_27": (4, 3, 22, (5, 22, "narrow", 3, 9)),
    "tall_32": (8, 4, 25, (7, 25, "narrow", 4, 8)),
    "tall_33": (8, 4, 26, (7, 26, "64bit", 5, 8)),
    "far_one_camera": (5, 8, "far", (11, 22, "64bit", 5, 8)),
    "full_32bit": (3, 3, 32, (5, 32, "64bit", 5, 8)),
    "saturated": (3, 3, "saturated", (5, "saturated", "64bit", 5, 8)),
}
# cases whose every single camera's frame is in a narrow plan while the tall frame is in the 64-bit layout
NARROW_SINGLES = ("tall_33", "far_one_camera")
FAR_KEY = 2 ** 21 + 4321  # depth key of the far Gaussian: 22 bits


def batch_plan_scene(name):
    """-> (H, W, C, T (tiles per frame), us [C,N,2], depths [C,N], areas [C,N,2], far (camera, row) or None)"""
    C, tb, db, _ = BATCH_PLANS[name]
    cams, far = [], None
    for c in range(C):
        H, W, T, (us, depths, areas) = key_plan_scene(tb, 14 if db == "far" else db, seed=1000 * c + 7 * tb + 1)
        if db == "far" and c == 2:
            sc = Scene()
            sc.add(us, depths, areas)
            far = (c, sc.one_patch(7, 9, depth_for_key([FAR_KEY])))
            sc.one_patch(7, 9, np.float32([1.0, 2.0, 3.0]))  # near Gaussians in the far one's tile
            us, depths, areas = sc.arrays()
        cams.append((us, depths, areas))
    return (H, W, C, T) + pad_cameras(cams) + (far,)


def camera_bins(H, W, us, depths, areas):
    """orc.bin of every camera on copies -> [(P, ranges, gsid, keys, depths culled, areas culled)]"""
    out = []
    for c in range(us.shape[0]):
        d, a = depths[c].copy(), areas[c].copy()
        out.append(orc.bin(H, W, us[c], d, a) + (d, a))
    return out


def tall_keys(bins, T):
    """the tall frame's keys from the per-camera oracle bins: tile id + c T in the tile field"""
    return np.concatenate([b[3] + (np.uint64(c * T) << np.uint64(32)) for c, b in enumerate(bins)])


@pytest.mark.parametrize("name", list(BATCH_PLANS))
def test_batch_plan_scenes_reach_their_plans(name):
    H, W, C, T, us, depths, areas, far = batch_plan_scene(name)
    want = BATCH_PLANS[name][3]
    bins = camera_bins(H, W, us, depths, areas)
    keys = tall_keys(bins, T)
    tb, db = widths(keys, C * T)
    dk = int((keys & np.uint64(0xFFFFFFFF)).max())
    p = key_plan(tall_height(C, H), W, dk)
    assert p["tbits"] == tb == want[0]
    assert (dk == 0xFFFFFFFF and want[1] == "saturated") or db == want[1], (db, want)
    assert plan_shape(p) == want[2:]
    singles = [key_plan(H, W, int((b[3] & np.uint64(0xFFFFFFFF)).max())) for b in bins]
    if name in NARROW_SINGLES:
        assert all(s["narrow"] for s in singles) and not p["narrow"]
    if far is not None:  # the 22-bit key is the far Gaussian's alone, in camera 2 alone
        c, row = far
        for k, b in enumerate(bins):
            dkc = b[3] & np.uint64(0xFFFFFFFF)
            assert int(dkc.max()).bit_length() == (22 if k == c else 14), k
        assert int(bins[c][3][np.flatnonzero(bins[c][2] == row)[0]] & np.uint64(0xFFFFFFFF)) == FAR_KEY
    assert all(b[0] > 0 for b in bins)


# ---------------------------------------------------------------- the tall frame's row limit
# (C, H, W): C gy = 65535 tile rows exactly; and C = 64 (GSB_BATCH_MAX_CAMERAS) at gy = 1023 with pad rows
ROW_LIMIT = [(3, 16 * 21845, 16), (64, 16 * 1023 - 5, 16)]


def row_limit_scene(C, H, W, seed):
    """Per camera: one-patch Gaussians in random tiles, on the first and the last tile row, straddling the
    frame's top and bottom edges, and huge ones reaching far past them (one past the whole tall frame), which
    only the clamp to the camera's own [0, gy] rows keeps out of its neighbours' tiles.
    -> dict of [C, N, ...] float32 / int32 arrays: us, cinv2ds, alphas, depths, colors, areas"""
    rng = np.random.default_rng(seed)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    cams = []
    for c in range(C):
        sc = Scene()
        sc.one_patch(rng.integers(0, gx, 120), rng.integers(0, gy, 120), rng.uniform(1, 30, 120), rng)
        sc.one_patch(rng.integers(0, gx, 8), gy - 1, rng.uniform(1, 30, 8), rng)  # the last tile row
        sc.one_patch(rng.integers(0, gx, 8), 0, rng.uniform(1, 30, 8), rng)       # the first
        sc.add([[W / 2, -6.0], [W / 3, -1.5]], [2.5, 3.5], (6, 12))                 # straddling the top edge
        sc.add([[W / 2, H + 4.0], [W / 3, H - 0.5]], [2.0, 4.0], (6, 12))           # and the bottom edge
        sc.add([[W / 2, H / 2]], 6.0, (W, 4 * C * H))                               # past the whole tall frame
        sc.add([[W / 2, H - 5.0]], 7.0, (4, 3 * H))                                 # three frames down
        sc.add([[W / 2, 5.0]], 8.0, (4, 2 * H))                                     # two frames up
        sc.add([[W / 2, H + 300.0], [W / 2, -300.0]], [9.0, 10.0], (4, 400))        # centred outside, reaching in
        cams.append(sc.arrays())
    us, depths, areas = pad_cameras(cams)
    N = us.shape[1]
    cinv = np.tile(np.float32([0.05, 0.01, 0.05]), (C, N, 1))
    return dict(us=us, cinv2ds=cinv, alphas=rng.uniform(0.05, 0.6, (C, N)).astype(np.float32), depths=depths,
                colors=rng.uniform(0, 1, (C, N, 3)).astype(np.float32), areas=areas)


@pytest.mark.parametrize("C,H,W", ROW_LIMIT)
def test_row_limit_scenes(C, H, W):
    gy = (H + 15) // 16
    assert C * gy == 65535 or (C, gy) == (64, 1023)
    assert tall_height(C, H) // 16 <= 65535
    s = row_limit_scene(C, H, W, seed=C)
    gx = (W + 15) // 16
    for c in (0, C - 1):
        d, a = s["depths"][c].copy(), s["areas"][c].copy()
        P, ranges, gsid, keys = orc.bin(H, W, s["us"][c], d, a)
        lens = ranges[:, 1] - ranges[:, 0]
        # the huge ones cover every tile; the first and last rows hold the edge Gaussians besides
        assert lens.min() >= 3 and lens[:gx].min() >= 5 and lens[-gx:].min() >= 5
        assert int(np.bincount(gsid).max()) == gx * gy


# ---------------------------------------------------------------- the batch capacity path
def capacity_scene(layout):
    """Three cameras; the last record (camera 2's last row) is a whole-frame Gaussian, so that the learnt
    patch count P ends exactly with it.  Batch A, then batch B in which one camera's depth keys need more bits
    than the plan learnt from A sorts.
    narrow: 64x40 frames (6 tall tile bits), depths 1-10 m (14-bit keys: a 20-bit key); in B camera 1 is 8
    times as far (17 bits).
    64bit: 320x235 frames (10 tall tile bits); camera 1 sees one Gaussian at 5000 m (23 bits: the 64-bit
    layout sorting 24 depth bits), which B moves to 16 777.3 m (25 bits, whose low 24 bits would sort it in
    front of the 1 m Gaussians of its tile).
    -> (H, W, us [C,N,2], depths A, depths B [C,N], areas [C,N,2])"""
    rng = np.random.default_rng(31 if layout == "narrow" else 32)
    H, W, k = (40, 64, 400) if layout == "narrow" else (235, 320, 1500)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    cams = []
    for c in range(3):
        sc = Scene()
        sc.one_patch(rng.integers(0, gx, k), rng.integers(0, gy, k), rng.uniform(1, 10, k), rng)
        if layout == "64bit" and c == 1:
            far = sc.one_patch(gx // 2, gy // 2, 5000.0)
            sc.one_patch(gx // 2, gy // 2, np.float32(1.0) + np.float32(0.001) * np.arange(8, dtype=np.float32))
        if c == 2:
            sc.add([[W / 2, H / 2]], 7.5, (W, H))
        cams.append(sc.arrays())
    us, dA, areas = pad_cameras(cams)
    dB = dA.copy()
    if layout == "narrow":
        dB[1] *= np.float32(8.0)
    else:
        dB[1, far] = 16777.3
    return H, W, us, dA, dB, areas


@pytest.mark.parametrize("layout", ["narrow", "64bit"])
def test_capacity_scenes(layout):
    H, W, us, dA, dB, areas = capacity_scene(layout)
    C, N = us.shape[:2]
    T = ((W + 15) // 16) * ((H + 15) // 16)
    bA, bB = camera_bins(H, W, us, dA, areas), camera_bins(H, W, us, dB, areas)
    kA, kB = tall_keys(bA, T), tall_keys(bB, T)
    dkA = int((kA & np.uint64(0xFFFFFFFF)).max())
    dkB = int((kB & np.uint64(0xFFFFFFFF)).max())
    pA = key_plan(tall_height(C, H), W, dkA)
    assert pA["narrow"] == (layout == "narrow")
    assert dkB.bit_length() > pA["depth_bits"]  # B's keys do not fit the plan learnt from A
    if layout == "64bit":
        assert pA["depth_bits"] == 24 and dkB.bit_length() == 25 and dkB % (1 << 24) < 1000
    # the whole-frame Gaussian is the last record with patches: it ends the patch list in data order
    assert np.bincount(bA[2][2]).argmax() == np.flatnonzero(dA[2] > 0).max()
    assert int(np.bincount(bA[2][2])[-1]) == T
