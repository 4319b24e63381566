"""GPU binning and sort (k_rects_scan, k_keys, the LSD radix passes, k_ranges) against the
oracle's binning, `oracle.bin`, on scenes built at the op surface so that every patch count,
tile rectangle and depth key is chosen rather than found by chance.

Every case asserts, bit for bit: the in-place culls, P, patch_range_per_tile and gsid_per_patch
of `splat` against the oracle; and the five outputs of the exact path (gsb_splat_bin +
gsb_splat_render) against the capacity path (gsb_splat_forward, bounds learnt from one frame).

The scenes reach every shape of sort `key_plan` can choose (1 to 4 passes of 8- or 9-bit digits
over 32-bit keys, key widths of exactly 32 and 33 bits, full 32-bit and saturated depth keys in
the 64-bit layout), sort sizes on both sides of the 4096-pair sort tile and of k_colscan's
2048-value span, key emission across k_rects_scan's 1024-Gaussian span, the capacity bounds
(P_cap == P, P_cap == P - 1, depth keys that outgrow a 64-bit plan) and the frames the binning
must refuse (2^30 patches, a patch count past 2^32, more than 65535 tiles in a row or column).
"""
import numpy as np
import pytest
import torch

from oracle import oracle as orc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def ops():
    from easygaussiansplatting_b200 import ops as o
    return o


@pytest.fixture(autouse=True)
def fresh_capacities():
    """each case learns its own capacity bounds"""
    ops()._CAPACITY.clear()
    yield
    ops()._CAPACITY.clear()


def t(a, dtype=torch.float32, device=DEV):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).to(device)


def n(x):
    return x.detach().cpu().numpy()


def bits(x):
    """a float32 / int32 tensor's bit patterns: NaN rows compare equal exactly when they are the same NaN"""
    return x.view(torch.int32)


def same(x, y):
    return torch.equal(bits(x), bits(y))


def need_free_memory(nbytes):
    free, total = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip("needs %.2f GB of free device memory, %.2f GB of %.2f GB free" % (
            nbytes / 2**30, free / 2**30, total / 2**30))


def depth_for_key(keys):
    """float32 depths whose depth key -- the float32 product depth * 1000 converted toward zero, as
    k_keys and the oracle compute it -- is exactly the given integer (every key below 2^22 has one;
    above, the float32 spacing skips some).  Raises ValueError for a key no depth reaches."""
    k = np.asarray(keys, dtype=np.float64).ravel()
    d0 = ((k + 0.5) / 1000.0).astype(np.float32)
    win = (d0.view(np.int32)[:, None] + np.arange(-64, 65, dtype=np.int32)).view(np.float32)  # +-64 ulps
    hit = np.floor((win * np.float32(1000.0)).astype(np.float64)) == k[:, None]
    if not hit.any(axis=1).all():
        raise ValueError("no float32 depth has depth key %d" % int(k[~hit.any(axis=1)][0]))
    return win[np.arange(len(k)), hit.argmax(axis=1)]


def top_bit_pair(d):
    """depths of two keys that differ only in bit d - 1, the larger first"""
    if d <= 22:
        return depth_for_key([201 + 2 ** (d - 1), 201])
    for a in range(2 ** 20, 2 ** 22, 256):  # above 2^24 the keys are float32 values: multiples of 256 near 2^31
        try:
            return depth_for_key([a + 2 ** (d - 1), a])
        except ValueError:
            pass
    raise AssertionError("no key pair differing in bit %d only" % (d - 1))


class Scene:
    """rows of (us, depth, areas) appended group by group; the row index is the Gaussian id"""

    def __init__(self):
        self.us, self.depths, self.areas = [], [], []

    def add(self, us, depths, areas):
        us = np.asarray(us, np.float64).reshape(-1, 2)
        k = len(us)
        self.us.append(us)
        self.depths.append(np.broadcast_to(np.asarray(depths, np.float32), (k,)))
        self.areas.append(np.broadcast_to(np.asarray(areas, np.int32), (k, 2)))
        return sum(len(u) for u in self.us) - k  # id of the first added row

    def one_patch(self, tx, ty, depths, rng=None):
        """Gaussians whose binning box is exactly tile (tx, ty) (area 1, mean inside [2, 14) of it)"""
        depths = np.atleast_1d(np.asarray(depths, np.float32))
        tx = np.broadcast_to(tx, depths.shape)
        ty = np.broadcast_to(ty, depths.shape)
        off = rng.uniform(2, 14, (len(depths), 2)) if rng is not None else np.full((len(depths), 2), 8.0)
        return self.add(np.stack([16.0 * tx + off[:, 0], 16.0 * ty + off[:, 1]], axis=1), depths, (1, 1))

    def arrays(self):
        return (np.ascontiguousarray(np.concatenate(self.us), np.float32),
                np.ascontiguousarray(np.concatenate(self.depths), np.float32),
                np.ascontiguousarray(np.concatenate(self.areas), np.int32))


def splat_inputs(us, depths, areas, seed=0, device=DEV):
    """device tensors of the splat op surface; conics, opacities and colours are filler"""
    N = len(depths)
    rng = np.random.default_rng(seed)
    cinv = np.tile(np.float32([0.05, 0.01, 0.05]), (N, 1))
    return (t(us, device=device), t(cinv, device=device),
            t(rng.uniform(0.05, 0.6, N).astype(np.float32), device=device), t(depths, device=device),
            t(rng.uniform(0, 1, (N, 3)).astype(np.float32), device=device),
            t(areas, torch.int32, device=device))


def run_splat(H, W, us, depths, areas, capacity=False, device=DEV):
    """-> (splat's five outputs, depths and areas after the in-place culls)"""
    u, ci, al, d, col, ar = splat_inputs(us, depths, areas, device=device)
    out = ops().splat(H, W, u, ci, al, d, col, ar, capacity=capacity)
    return out, d, ar


def check_binning(H, W, us, depths, areas, capacity=True):
    """bit-exact against oracle.bin; then the capacity path (one learning frame, one frame on the
    learnt bounds, which must not be redone) bit-identical to the exact path.
    -> the oracle's (P, ranges, gsid, keys)"""
    o = ops()
    d_or, a_or = depths.copy(), areas.copy()
    P, ranges, gsid, keys = orc.bin(H, W, us, d_or, a_or)
    exact, d, a = run_splat(H, W, us, depths, areas)
    assert np.array_equal(n(bits(d)), d_or.view(np.int32)), "in-place depth cull differs"
    assert np.array_equal(n(a), a_or), "in-place areas cull differs"
    assert exact[4].numel() == P, (exact[4].numel(), P)
    assert np.array_equal(n(exact[3]), ranges), "patch_range_per_tile differs"
    assert np.array_equal(n(exact[4]), gsid), "gsid_per_patch (sort order) differs"
    if capacity and P > 0:
        run_splat(H, W, us, depths, areas, capacity=True)  # learns the bounds (exact path)
        assert (0, H, W, len(depths)) in o._CAPACITY
        before = dict(o.CAPACITY_STATS)
        cap, d2, a2 = run_splat(H, W, us, depths, areas, capacity=True)
        assert o.CAPACITY_STATS["capacity_frames"] == before["capacity_frames"] + 1, "frame was redone"
        assert o.CAPACITY_STATS["outgrown"] == before["outgrown"]
        for name, x, y in zip(("image", "contrib", "final_tau", "ranges", "gsid"), exact, cap):
            assert same(x, y), "capacity path differs from the exact path: " + name
        assert same(d, d2) and same(a, a2)
    torch.cuda.synchronize()
    return P, ranges, gsid, keys


def widths(keys, T):
    """(tile bits, depth-key bits) the scene needs, from the oracle's 64-bit keys"""
    return (T - 1).bit_length(), int((keys & np.uint64(0xFFFFFFFF)).max()).bit_length()


# ---------------------------------------------------------------- 1. every key plan
# (tile bits, depth-key bits): tile + depth = 8, 9, 16, 17, 24, 25, 27, 28, 32 (a 32-bit key using
# every bit) and 33 (the smallest 64-bit key); then 32-bit depth keys and saturated ones.
PLANS = [(0, 8), (1, 8), (4, 12), (5, 12), (8, 16), (9, 16), (10, 17), (11, 17), (12, 20), (12, 21),
         (4, 32), (4, "saturated")]


def key_plan_scene(tbits, dbits, seed):
    rng = np.random.default_rng(seed)
    sat = dbits == "saturated"
    d = 32 if sat else dbits
    gx, gy = 2 ** ((tbits + 1) // 2), 2 ** (tbits // 2)
    T = gx * gy
    tiles = sorted({0, T // 2, T - 1})
    tile_xy = lambda i: (i % gx, i // gx)
    sc = Scene()

    def filler(k):
        """k one-patch Gaussians in random tiles with random depth keys of at most d bits"""
        hi = (2.0 ** d - 2) / 1000.0 * 0.999
        dep = rng.uniform(0.2, hi, k).astype(np.float32)
        sc.one_patch(rng.integers(0, gx, k), rng.integers(0, gy, k), dep, rng)

    filler(300)
    for ti in tiles:
        tx, ty = tile_xy(ti)
        # differ only in bit 0 (the larger key first: the sort has to swap them), at both ends of the range
        sc.one_patch(tx, ty, depth_for_key([201, 200]))
        if d <= 22:
            sc.one_patch(tx, ty, depth_for_key([2 ** d - 1, 2 ** d - 2]))
        # differ only in the highest depth-key bit (no such pair with 8 bits: keys start at 200)
        if d > 8:
            sc.one_patch(tx, ty, top_bit_pair(d))
        filler(50)
    # 9000 Gaussians in one tile, every other one on the same key: ties spread over three sort
    # tiles and interleaved with other keys; a second tied run in the last tile
    tx, ty = tile_xy(T // 2)
    if sat:  # different depths, one key: all saturate to 0xffffffff
        tie = np.tile(np.float32([np.inf, 4.295e6, 5e6, 1e30]), 1125)
    else:
        tie = np.full(4500, (2.0 ** d - 1 - 0.2 * 2.0 ** (d - 1)) / 1000.0, np.float32)
    other = rng.uniform(0.2, (2.0 ** d - 2) / 1000.0 * 0.999, len(tie)).astype(np.float32)
    mixed = np.empty(2 * len(tie), np.float32)
    mixed[0::2], mixed[1::2] = tie, other
    sc.one_patch(tx, ty, mixed)
    filler(200)
    tx, ty = tile_xy(T - 1)
    sc.one_patch(tx, ty, np.concatenate([tie[:700], other[:300]]))
    # NaN depth: binned with depth key 0; NaN / +-inf means: culled in place
    for du in ((np.nan, 8.0), (8.0, np.nan), (np.inf, 8.0), (-np.inf, 8.0), (8.0, np.inf), (np.nan, np.nan)):
        sc.add([du], 5.0, (2, 2))
        sc.one_patch(0, 0, np.float32(np.nan))
    filler(200)
    return 16 * gy, 16 * gx, T, sc.arrays()


@pytest.mark.parametrize("tbits,dbits", PLANS)
def test_every_key_plan(tbits, dbits):
    H, W, T, (us, depths, areas) = key_plan_scene(tbits, dbits, seed=tbits * 100 + (dbits if dbits != "saturated" else 99))
    P, ranges, gsid, keys = check_binning(H, W, us, depths, areas)
    tb, db = widths(keys, T)
    assert tb == tbits and P > 8192
    if dbits == "saturated":
        assert (keys & np.uint64(0xFFFFFFFF)).max() == 0xFFFFFFFF
        assert ((keys & np.uint64(0xFFFFFFFF)) == 0xFFFFFFFF).sum() >= 4500
    else:
        assert db == dbits, (db, dbits)
    # the NaN-depth rows were binned with depth key 0: first in tile 0
    nan_rows = np.flatnonzero(np.isnan(depths))
    assert np.array_equal(gsid[:len(nan_rows)], nan_rows)


# ---------------------------------------------------------------- 2. sort sizes and digit skew
SIZES = [1, 4095, 4096, 4097, 8192, 12289, 16384, 16385, 32768, 32769]
# one tile (depth keys of 24 bits: three 8-bit passes) and two tiles (1 + 16 bits: two 9-bit
# passes); a pass over 8 or more sort tiles of 8-bit digits, or 4 or more of 9-bit digits, scans
# more than one k_colscan span
FRAMES = {"1tile": (16, 16, 24), "2tiles": (16, 32, 16)}


def sort_scene(frame, P, pattern):
    """P one-patch Gaussians, all in one tile or alternating between two, whose depth keys all
    have the frame's width (their top bit set)"""
    H, W, d = FRAMES[frame]
    two = W == 32
    i = np.arange(P)
    lo, hi = 2.0 ** (d - 1) / 1000.0, (2.0 ** d - 1) / 1000.0  # depths of the key range
    if pattern == "equal":
        depths = np.full(P, 0.7 * lo + 0.3 * hi, np.float32)
    elif pattern == "decreasing":  # strictly decreasing in id within each tile
        depths = (depth_for_key(2 ** (d - 1) + (P - 1 - i) // 2) if two
                  else (lo + 1.0 + 0.01 * (P - 1 - i)).astype(np.float32))  # (keys 10 apart)
    elif pattern == "three":
        depths = np.float32([lo + 0.5, 0.5 * (lo + hi), hi - 0.5])[(i * 7 + i // 5) % 3]
    else:
        depths = np.random.default_rng(P).uniform(lo, hi, P).astype(np.float32)
    tx = i % 2 if two else np.zeros(P, np.int64)
    us = np.stack([16.0 * tx + 8.0, np.full(P, 8.0)], axis=1).astype(np.float32)
    return H, W, us, depths, np.ones((P, 2), np.int32)


@pytest.mark.parametrize("pattern", ["equal", "decreasing", "three", "random"])
@pytest.mark.parametrize("frame", list(FRAMES))
@pytest.mark.parametrize("P", SIZES)
def test_sort_sizes_and_digit_skew(P, frame, pattern):
    H, W, us, depths, areas = sort_scene(frame, P, pattern)
    Pr, ranges, gsid, keys = check_binning(H, W, us, depths, areas)
    assert Pr == P
    i = np.arange(P)
    per_tile = [i[i % 2 == 0], i[i % 2 == 1]] if W == 32 else [i]
    if pattern == "equal":  # every key of a sort tile has the same digit in every pass
        assert np.array_equal(gsid, np.concatenate(per_tile))
    elif pattern == "decreasing":
        assert np.array_equal(gsid, np.concatenate([p[::-1] for p in per_tile]))
    elif pattern == "three":  # a stable partition
        dk = keys & np.uint64(0xFFFFFFFF)
        assert len(np.unique(dk)) == min(P, 3)
        tile = (keys >> np.uint64(32)).astype(np.int64)
        want = np.lexsort((gsid, dk, tile))
        assert np.array_equal(want, np.arange(P)) and np.all(np.diff(tile) >= 0)
    tb, db = widths(keys, (W // 16) * (H // 16))
    assert tb + db == (24 if W == 16 else 17), (tb, db)


# ---------------------------------------------------------------- 3. key emission
def emission_scene(N, seed):
    """80 x 48 tiles.  Per warp of 32 consecutive Gaussians: whole-frame Gaussians in lane 0 (every
    8th warp) or lane 31 (every 8th, offset 4), otherwise a mix of one-patch Gaussians, 1-tile-wide
    columns over the full height and single-row rectangles 65 tiles wide; every 16th pair of warps
    is culled whole (64 consecutive Gaussians: half by depth, half in place by an empty rectangle)."""
    gx, gy = 80, 48
    W, H = 16 * gx, 16 * gy
    rng = np.random.default_rng(seed)
    i = np.arange(N)
    warp, lane = i // 32, i % 32
    kind = rng.integers(0, 3, N)
    tx, ty = rng.integers(0, gx, N), rng.integers(0, gy, N)
    us = np.stack([16.0 * tx + rng.uniform(2, 14, N), 16.0 * ty + rng.uniform(2, 14, N)], axis=1)
    areas = np.ones((N, 2), np.int32)
    col = kind == 1
    us[col] = np.stack([16.0 * tx[col] + 8, np.full(col.sum(), H / 2)], axis=1)
    areas[col] = (2, H)
    row = kind == 2
    a = rng.integers(0, gx - 65 + 1, row.sum())
    us[row] = np.stack([16.0 * a + 520, 16.0 * ty[row] + 8], axis=1)
    areas[row] = (516, 2)
    whole = ((warp % 8 == 0) & (lane == 0)) | ((warp % 8 == 4) & (lane == 31))
    us[whole] = (W / 2, H / 2)
    areas[whole] = (W, H)
    depths = np.round(rng.uniform(1.0, 50.0, N), 2).astype(np.float32)  # many exact ties
    culled = (warp % 16 == 6) | (warp % 16 == 7)
    depths[culled & (warp % 16 == 6)] = -1.0
    us[culled & (warp % 16 == 7)] = (-1000.0, -1000.0)
    return H, W, us.astype(np.float32), depths, areas, dict(whole=whole, col=col & ~whole & ~culled,
                                                           row=row & ~whole & ~culled, culled=culled)


@pytest.mark.parametrize("N", [1023, 1024, 1025, 32 * 1024 + 1])
def test_key_emission_mixed_warps(N):
    H, W, us, depths, areas, kinds = emission_scene(N, seed=N)
    d_in = depths.copy()
    P, ranges, gsid, keys = check_binning(H, W, us, depths, areas)
    counts = np.bincount(gsid, minlength=N)
    T = (W // 16) * (H // 16)
    assert (counts[kinds["whole"]] == T).all() and kinds["whole"].sum() >= 1
    assert (counts[kinds["col"]] == H // 16).all() and (counts[kinds["row"]] == 65).all()
    assert (counts[kinds["culled"]] == 0).all()
    assert (d_in[kinds["culled"]] >= 0).any()  # (half of the culled rows are culled in place)


# ---------------------------------------------------------------- 4. capacity bounds
def test_capacity_exactly_P_and_one_short():
    """P_cap == P: the last Gaussian (whole-frame, 3840 patches) ends exactly at the capacity, and
    the frame is served without a redo; P_cap == P - 1: it is redone, with the same outputs"""
    o = ops()
    N = 1025
    H, W, us, depths, areas, _ = emission_scene(N, seed=3)
    us[-1], areas[-1], depths[-1] = (W / 2, H / 2), (W, H), 7.5
    P, ranges, gsid, keys = check_binning(H, W, us, depths, areas, capacity=False)
    exact, _, _ = run_splat(H, W, us, depths, areas)
    dk_cap = o._next_capacity(P, int((keys & np.uint64(0xFFFFFFFF)).max()))[1]
    for P_cap, redo in ((P, False), (P - 1, True)):
        o._CAPACITY[(0, H, W, N)] = (P_cap, dk_cap)
        before = dict(o.CAPACITY_STATS)
        out, _, _ = run_splat(H, W, us, depths, areas, capacity=True)
        assert o.CAPACITY_STATS["outgrown"] == before["outgrown"] + int(redo), P_cap
        assert o.CAPACITY_STATS["capacity_frames"] == before["capacity_frames"] + int(not redo), P_cap
        for x, y in zip(exact, out):
            assert same(x, y), P_cap
    torch.cuda.synchronize()


def far_gaussian_frames():
    """1080p (13 tile bits).  Frame A: 6000 one-patch Gaussians at 1-10 m, one of them (id 3000) at
    600 m: depth keys of 20 bits, so the next frame's plan is the 64-bit layout with 24 depth bits
    sorted.  Frame B: the same Gaussian at 16 777.3 m, whose depth key needs 25 bits; its tile also
    holds Gaussians at 1 m, in front of which its low 24 bits (= 84) would sort it."""
    rng = np.random.default_rng(21)
    W, H = 1920, 1080
    sc = Scene()
    sc.one_patch(rng.integers(0, 120, 3000), rng.integers(0, 67, 3000), rng.uniform(1, 10, 3000), rng)
    far = sc.one_patch(60, 30, 600.0)
    sc.one_patch(60, 30, np.full(8, 1.0, np.float32) + np.float32(0.001) * np.arange(8))
    sc.one_patch(rng.integers(0, 120, 2991), rng.integers(0, 67, 2991), rng.uniform(1, 10, 2991), rng)
    us, dA, areas = sc.arrays()
    dB = dA.copy()
    dB[far] = 16777.3
    return H, W, us, dA, dB, areas, far


def test_capacity_depth_keys_outgrow_64bit_plan():
    o = ops()
    H, W, us, dA, dB, areas, far = far_gaussian_frames()
    N = len(dA)
    PB, ranges, gsid, keys = orc.bin(H, W, us, dB.copy(), areas.copy())
    dk = keys & np.uint64(0xFFFFFFFF)
    assert int(dk.max()).bit_length() == 25 and int(dk.max()) % (1 << 24) < 1000
    exactB, _, _ = run_splat(H, W, us, dB, areas)
    assert np.array_equal(n(exactB[4]), gsid) and np.array_equal(n(exactB[3]), ranges)
    run_splat(H, W, us, dA, areas, capacity=True)  # learns from frame A
    assert o._CAPACITY[(0, H, W, N)][1] == (1 << 20) - 1
    before = dict(o.CAPACITY_STATS)
    outB, _, _ = run_splat(H, W, us, dB, areas, capacity=True)
    torch.cuda.synchronize()
    for name, x, y in zip(("image", "contrib", "final_tau", "ranges", "gsid"), exactB, outB):
        assert same(x, y), "capacity path mis-sorted the far Gaussian: " + name
    assert o.CAPACITY_STATS["outgrown"] == before["outgrown"] + 1


def test_graphed_step_depth_keys_outgrow_64bit_plan():
    """the same defect through the captured training step: moving one parameter row from 600 m to
    16 777.3 m (same pixel, same footprint) must make backward() raise CapacityError"""
    from easygaussiansplatting_b200.graphed import CapacityError, GraphedFusedStep
    from easygaussiansplatting_b200.gsfunction import Camera
    from easygaussiansplatting_b200.scene import synthetic_scene
    W, H, N = 1920, 1080, 20000
    sc = synthetic_scene(N, W, H, sh_dim=3, seed=8)
    u = sc["pws"][:, 0] / sc["pws"][:, 2] * sc["fx"] + sc["cx"]
    v = sc["pws"][:, 1] / sc["pws"][:, 2] * sc["fy"] + sc["cy"]
    near = np.flatnonzero((u > 300) & (u < W - 300) & (v > 200) & (v < H - 200))[:2]
    j, f = int(near[0]), int(near[1])

    def place(z):
        s = z / sc["pws"][j, 2]
        return t(sc["pws"][j] * s), t(sc["scales"][j] * s)

    P = {k: t(sc[k]) for k in ("pws", "shs", "scales", "rots")}
    al = t(sc["alphas"][:, None])
    P["pws"][f], P["scales"][f] = place(600.0)
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]))
    step = GraphedFusedStep(P["pws"], P["shs"], al, P["scales"], P["rots"], cam)
    assert step.dk_cap == (1 << 20) - 1
    step.forward()
    step.backward()  # within the learnt bounds
    with torch.no_grad():
        P["pws"][f], P["scales"][f] = place(16777.3)
    step.forward()
    torch.cuda.synchronize()
    with pytest.raises(CapacityError):
        step.backward()


# ---------------------------------------------------------------- 5. refusals
def whole_frame(N, W, H):
    us = np.tile(np.float32([W / 2, H / 2]), (N, 1))
    return us, np.full(N, 3.0, np.float32), np.tile(np.int32([W, H]), (N, 1))


@pytest.mark.parametrize("N,what", [(131_600, "2^30"), (526_400, "2^32")])
def test_refuse_too_many_patches(N, what):
    """131 600 (526 400) Gaussians each covering all 8160 tiles of a 1080p frame: 1.07e9 patches
    (past 2^30), resp. 4.2954e9 (past 2^32: k_rects_scan's saturating flag).  Both paths raise;
    the capacity path after a small learning frame of the same N."""
    o = ops()
    W, H = 1920, 1080
    need_free_memory(256 << 20)
    us, depths, areas = whole_frame(N, W, H)
    with pytest.raises(RuntimeError, match="2\\^30 patches"):
        run_splat(H, W, us, depths, areas)
    torch.cuda.synchronize()
    rng = np.random.default_rng(5)
    small = np.stack([rng.uniform(0, W, N), rng.uniform(0, H, N)], axis=1).astype(np.float32)
    run_splat(H, W, small, depths, np.ones((N, 2), np.int32), capacity=True)  # learns small bounds
    assert o._CAPACITY[(0, H, W, N)][0] < 1 << 30
    with pytest.raises(RuntimeError, match="2\\^30 patches"):
        run_splat(H, W, us, depths, areas, capacity=True)
    torch.cuda.synchronize()


def edge_grid_scene(long_tiles, tall):
    """65535 x 2 tiles (or 2 x 65535): one-patch Gaussians in the last column (last row) of both
    tile rows, a 2-tile-high column there, a 65-tile row ending there, a whole-frame Gaussian, one
    reaching past the edge, and random one-patch Gaussians along the strip"""
    rng = np.random.default_rng(long_tiles)
    last = long_tiles - 1
    sc = Scene()
    sc.one_patch(rng.integers(0, long_tiles, 3000), rng.integers(0, 2, 3000), rng.uniform(1, 30, 3000), rng)
    sc.one_patch([last, last, last], [0, 1, 0], [2.0, 3.0, 1.5], rng)
    sc.add([16.0 * last + 8, 16.0], 4.0, (2, 16))                    # both tile rows of the last column
    sc.add([16.0 * (last - 65 + 1) + 520, 8.0], 2.5, (516, 2))       # tiles last-64 .. last of row 0
    sc.add([16.0 * long_tiles / 2, 16.0], 9.0, (16 * long_tiles, 32))  # the whole frame
    sc.add([16.0 * long_tiles + 40, 24.0], 1.2, (60, 2))             # clipped at the edge, row 1
    sc.one_patch(rng.integers(long_tiles - 100, long_tiles, 500), rng.integers(0, 2, 500), rng.uniform(1, 30, 500), rng)
    us, depths, areas = sc.arrays()
    if tall:
        us, areas = np.ascontiguousarray(us[:, ::-1]), np.ascontiguousarray(areas[:, ::-1])
    return us, depths, areas


@pytest.mark.parametrize("tall", [False, True], ids=["wide", "tall"])
def test_grid_limit(tall):
    """65535 tiles in a row (column) bin exactly; 65536 are refused by both paths instead of
    wrapping the 16-bit rectangle bound to 0"""
    o = ops()
    need_free_memory(3 << 30)
    L = 65535 * 16
    H, W = (L, 32) if tall else (32, L)
    us, depths, areas = edge_grid_scene(65535, tall)
    P, ranges, gsid, keys = check_binning(H, W, us, depths, areas)
    T = ranges.shape[0]
    assert T == 2 * 65535
    last = [65534, 2 * 65535 - 1] if not tall else [2 * 65534, 2 * 65534 + 1]
    assert all(ranges[i, 1] - ranges[i, 0] >= 4 for i in last)
    H2, W2 = (L + 16, 32) if tall else (32, L + 16)
    us2, depths2, areas2 = edge_grid_scene(65536, tall)
    with pytest.raises(RuntimeError, match="65535 tiles"):
        run_splat(H2, W2, us2, depths2, areas2)
    o._CAPACITY[(0, H2, W2, len(depths2))] = (1 << 20, (1 << 20) - 1)
    with pytest.raises(RuntimeError, match="65535 tiles"):
        run_splat(H2, W2, us2, depths2, areas2, capacity=True)
    torch.cuda.synchronize()


# ---------------------------------------------------------------- 6. a second device
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two CUDA devices")
def test_64bit_keys_on_second_device():
    """k_radix_pass needs its shared-memory opt-in on every device it runs on: a 64-bit-key frame
    on device 0, then the same frame on device 1, bit-identical to each other and to the oracle"""
    H, W, T, (us, depths, areas) = key_plan_scene(12, 21, seed=4)
    P, ranges, gsid, keys = orc.bin(H, W, us, depths.copy(), areas.copy())
    outs = []
    for dev in ("cuda:0", "cuda:1"):
        out, _, _ = run_splat(H, W, us, depths, areas, device=dev)
        torch.cuda.synchronize(dev)
        assert np.array_equal(n(out[4]), gsid) and np.array_equal(n(out[3]), ranges), dev
        outs.append([x.cpu() for x in out])
    for x, y in zip(*outs):
        assert same(x, y)
