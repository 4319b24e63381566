"""Batched 2D Gaussian Splatting (DESIGN 3.25) at its edges, on the host: the scene builders of
test_gpu_surfel_batch_edges.py checked with the fp64 surfel oracle (`so.preprocess`, `so.bin_f32`) and the
`key_plan` / `tall_height` mirror of test_batch_edges_cpu.py to reach what each is built for.  A builder
that misses its target fails here, not silently on the GPU.

- PLAN_BATCHES: surfel batches whose tall frame sorts with each key plan the 3DGS batch reaches (one to
  three passes of 9-bit digits, four of 8 bits, the 64-bit layout with 26-bit, 32-bit and saturated
  depth keys), one of them with every single frame in a narrow plan; the tall frame's tile rows and the
  plan the capacity path sizes its sort for.
- special_batch: test_surfel_edge_scenes_cpu.special_scene seen by seven cameras, so that each special
  surfel is degenerate, capped or culled in some of them and ordinary in others; one camera turned away.
- boundary_batch: surfels across the bottom edge of every frame and on the first row below it.

A camera is a dict of fp32 values (Rcw [3,3], tcw, twc, fx, fy, cx, cy): what the kernels read."""
import numpy as np
import pytest

from oracle import surfel_oracle as so

from test_batch_edges_cpu import key_plan, plan_shape, tall_height, tall_keys
from test_surfel_edge_scenes_cpu import camera, cull_box, fronto, quat, rot, special_scene

f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)


# ---------------------------------------------------------------- cameras and scenes
def make_camera(Rcw, twc, fx, fy, cx, cy):
    """fp32 camera with tcw = -Rcw twc (computed in fp64 from the fp32 Rcw, twc)"""
    R, tw = f32(Rcw), f32(twc)
    tc = f32(-R.astype(np.float64) @ tw.astype(np.float64))
    return dict(Rcw=R, tcw=tc, twc=tw, fx=float(np.float32(fx)), fy=float(np.float32(fy)), cx=float(np.float32(cx)),
                cy=float(np.float32(cy)))


def jittered_cameras(C, W, H, f, seed, ang=0.01, shift=0.05):
    """C cameras a small rotation (about `ang` rad) and shift apart around the identity pose, with
    intrinsics of their own; camera 0 is the identity"""
    rng = np.random.default_rng(seed)
    cams = []
    for c in range(C):
        R = np.eye(3) if c == 0 else rot(rng.normal(size=3), ang * rng.uniform(0.5, 1.0))
        tw = np.zeros(3) if c == 0 else rng.normal(size=3) * shift
        fx = f * (1.0 + 0.02 * c)
        cams.append(make_camera(R, tw, fx, fx * 1.01, W / 2 - 0.3 + 0.37 * c, H / 2 + 0.2 - 0.23 * c))
    return cams


def to_world(pc, Rc, cam):
    """camera-frame centres and rotations (columns R e0, R e1, R e2) of `cam` -> pws, rots (fp64)"""
    Rcw, tcw = cam["Rcw"].astype(np.float64), cam["tcw"].astype(np.float64)
    return (np.asarray(pc, np.float64) - tcw) @ Rcw, np.stack([quat(Rcw.T @ R) for R in Rc])


def scene_dict(pws, rots, scales, shs, alphas):
    return dict(pws=f32(pws), rots=f32(rots), scales=f32(scales), shs=f32(shs), alphas=f32(alphas))


def pre_cam(s, cam):
    """the fp64 oracle's per-surfel stages of scene s in camera cam"""
    return so.preprocess(s["pws"], s["rots"], s["scales"], s["shs"], cam["Rcw"], cam["tcw"], cam["twc"], cam["fx"],
                         cam["fy"], cam["cx"], cam["cy"])


def disks(rng, cam, W, H, N, z, sigma=(0.8, 4.0), margin=2.0, log_depth=False):
    """N disks over camera cam's frame: centres at pixels inside [margin, W - margin] x [margin, H - margin],
    camera depths in z (log-uniform if log_depth), sigma in pixels, tilted up to 40 degrees from
    fronto-parallel -> (camera-frame centres, rotations, disk scales [N,3])"""
    x, y = rng.uniform(margin, W - margin, N), rng.uniform(margin, H - margin, N)
    zz = np.exp(rng.uniform(np.log(z[0]), np.log(z[1]), N)) if log_depth else rng.uniform(*z, N)
    pc = np.stack([(x - cam["cx"]) * zz / cam["fx"], (y - cam["cy"]) * zz / cam["fy"], zz], 1)
    Rc = [rot(rng.normal(size=3), rng.uniform(0, 0.7)) @ fronto(1)[0] for _ in range(N)]
    sg = rng.uniform(*sigma, (N, 2)) * zz[:, None] / cam["fx"]
    return pc, Rc, np.concatenate([sg, rng.uniform(0, 0.05, (N, 1)) * zz[:, None]], 1)


def build(rng, parts, cam, k):
    """parts: [(centres, rotations, scales, alphas)] in cam's frame -> scene dict with SH degree k"""
    pc = np.concatenate([p[0] for p in parts])
    Rc = [R for p in parts for R in p[1]]
    scales = np.concatenate([p[2] for p in parts])
    alphas = np.concatenate([np.broadcast_to(p[3], (len(p[0]),)) for p in parts])
    pws, rots = to_world(pc, Rc, cam)
    return scene_dict(pws, rots, scales, rng.normal(scale=0.3, size=(len(pc), 3 * k)), alphas)


# ---------------------------------------------------------------- the tall frame's key plans
# name -> (C, W, H, camera depths of the random disks, depth of the two far disks, focal length,
# camera jitter (rad, m); what the tall frame reaches: (tile bits, depth-key bits, layout, passes,
# digit bits)).  The far disks are at the frame's centre in every camera and set the largest depth key.
PLAN_BATCHES = {
    "tall_9": (2, 13, 11, (0.205, 0.24), 0.245, 20.0, (0.005, 0.001), (1, 8, "narrow", 1, 9)),
    "tall_18": (3, 13, 11, (2.0, 30.0), 50.0, 20.0, (0.01, 0.05), (2, 16, "narrow", 2, 9)),
    "tall_25": (4, 29, 13, (2.0, 1500.0), 3000.0, 25.0, (0.01, 0.05), (3, 22, "narrow", 3, 9)),
    "tall_32": (8, 61, 63, (2.0, 12000.0), 25000.0, 50.0, (0.005, 0.05), (7, 25, "narrow", 4, 8)),
    "tall_33": (8, 61, 63, (2.0, 12000.0), 50000.0, 50.0, (0.005, 0.05), (7, 26, "64bit", 5, 8)),
    "saturated": (3, 45, 29, (2.0, 60.0), 6.0e6, 40.0, (0.005, 0.05), (5, "saturated", "64bit", 5, 8)),
}
NARROW_SINGLES = ("tall_33",)  # every single frame sorts 32-bit keys, the tall frame 64-bit ones


def plan_batch(name, k=1):
    """-> (W, H, cams, scene): 240 random disks (saturated: also two at 3e6 m, whose depth keys have
    32 bits) and two far ones at the frame's centre, seen by C jittered cameras"""
    C, W, H, z, zfar, f, (ang, shift), _ = PLAN_BATCHES[name]
    rng = np.random.default_rng(len(name) * 7 + C)
    cams = jittered_cameras(C, W, H, f, seed=C + W, ang=ang, shift=shift * z[0])
    cam = cams[0]
    parts = [disks(rng, cam, W, H, 240, z, log_depth=True) + (rng.uniform(0.1, 0.95, 240),)]
    for zf in ((3.0e6, zfar) if name == "saturated" else (zfar,)):
        pc, Rc, sc = disks(rng, cam, W, H, 2, (zf, zf * 1.0001), sigma=(2.0, 3.0), margin=0.0)
        pc[:, 0], pc[:, 1] = (np.array([0.4, 0.6]) * W - cam["cx"]) * pc[:, 2] / cam["fx"], \
            (np.array([0.45, 0.55]) * H - cam["cy"]) * pc[:, 2] / cam["fy"]
        parts.append((pc, Rc, sc, 0.8))
    return W, H, cams, build(rng, parts, cam, k)


def camera_bins(W, H, s, cams):
    """the oracle's binning of every camera on its own fp32 (u, depth, area) -> [(P, ranges, gsid, keys)]"""
    return [so.bin_f32(H, W, pre_cam(s, cam)) for cam in cams]


def depth_key_max(keys):
    return int((keys & np.uint64(0xFFFFFFFF)).max(initial=0))


@pytest.mark.parametrize("name", list(PLAN_BATCHES))
def test_plan_batches_reach_their_plans(name):
    C, W, H, *_, want = PLAN_BATCHES[name]
    _, _, cams, s = plan_batch(name)
    T = ((W + 15) // 16) * ((H + 15) // 16)
    bins = camera_bins(W, H, s, cams)
    assert all(b[0] > 0 for b in bins)
    keys = tall_keys(bins, T)
    dk = depth_key_max(keys)
    p = key_plan(tall_height(C, H), W, dk)
    assert p["tbits"] == want[0] and plan_shape(p) == want[2:], (p, want)
    assert (want[1] == "saturated" and dk == 0xFFFFFFFF) or p["dbits"] == want[1], (dk, want)
    # the tall frame's tile rows: C frames of gy rows, pad rows below every frame with a partial tile row
    assert tall_height(C, H) // 16 == C * ((H + 15) // 16) and (H % 16 != 0 or W % 16 != 0)
    # the capacity path sizes its sort for the key width of the largest depth key it saw: the same plan
    from easygaussiansplatting_b200.ops import _next_capacity
    assert plan_shape(key_plan(tall_height(C, H), W, _next_capacity(1, dk)[1])) == plan_shape(p)
    singles = [key_plan(H, W, depth_key_max(b[3])) for b in bins]
    if name in NARROW_SINGLES:
        assert all(q["narrow"] for q in singles) and not p["narrow"]
    if name == "saturated":  # 32-bit and saturated depth keys in every camera
        for b in bins:
            d = b[3] & np.uint64(0xFFFFFFFF)
            assert (d == 0xFFFFFFFF).sum() >= 2 and ((d >= 2 ** 31) & (d < 0xFFFFFFFF)).sum() >= 2
    # the far disks are drawn in every camera and hold its largest key (its 2^(bits - 1) bit set)
    far = len(s["pws"]) - 2
    for b in bins:
        assert np.isin([far, far + 1], b[2]).all()
        assert depth_key_max(b[3]).bit_length() == depth_key_max(keys).bit_length()


# ---------------------------------------------------------------- degenerate in one camera
KINDS = ("ordinary", "culled", "alpha-culled", "capped", "unbounded", "edge-on", "grazing", "sub-pixel", "needle",
         "frame-sized", "off-screen", "flipped")


def special_cameras():
    """seven cameras around special_scene's posed_b: 0 posed_b itself, 1 posed_b turned around (every
    surfel behind it), 2-5 moved and turned so that the view rays, depths and distances change"""
    W, H = 96, 64
    Rb, _, twb = camera("posed_b")
    f, cx, cy = 0.8 * W, W / 2 - 0.3, H / 2 + 0.2
    cams = [make_camera(Rb, twb, f, f, cx, cy), make_camera(np.diag([-1.0, 1.0, -1.0]) @ Rb, twb, f, f, cx, cy)]
    # camera-frame moves of posed_b: (rotation about the camera axes, centre offset in the camera frame, focal)
    moves = [(rot([0, 1, 0], 0.35), [1.2, 0.0, 0.3], f), (rot([1, 0, 0], -0.3), [0.0, -1.0, -0.4], f),
             (np.eye(3), [0.0, 0.0, -40.0], 10 * f), (rot([0.3, 1, 0.2], -0.5), [-1.6, 0.5, 0.8], 0.8 * f)]
    for R, off, fc in moves:
        Rcw = R.T @ Rb
        twc = twb + Rb.T @ np.asarray(off, np.float64)
        cams.append(make_camera(Rcw, twc, fc, fc * 1.02, cx + 1.3, cy - 0.7))
    # 6: posed_b's orientation 0.75 m in front of the sub-pixel disk (2) at 3 f, its principal point
    # moved so that the disk is at the frame's centre: 1.2 px
    p2 = np.array([(12.4 - cx) * 5.0005 / f, (50.3 - cy) * 5.0005 / f, 5.0005])
    cams.append(make_camera(Rb, twb + Rb.T @ (p2 * (1 - 0.75 / 5.0005)), 3 * f, 3 * f, W / 2 - 3 * (12.4 - cx),
                            H / 2 - 3 * (50.3 - cy)))
    return W, H, cams


def special_batch(k=4):
    """-> (W, H, cams, scene): special_scene at posed_b and the seven cameras of special_cameras"""
    sc = special_scene(k=k, cam="posed_b")
    W, H, cams = special_cameras()
    return W, H, cams, scene_dict(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["alphas"])


def kinds_in(s, cam, W, H):
    """the kind (KINDS) of every surfel of s in cam, from the fp64 oracle, the first that applies:
    culled (behind the camera or an unbounded footprint), alpha-culled (alpha < 0.002: a -inf cull box),
    capped (a binning half-extent at 2^24), unbounded (a +inf cull box), edge-on (the normal within 3
    degrees of across the view ray), grazing (within 10), sub-pixel (both axes under 0.3 px at the
    centre), needle (axes over 20:1 on screen), frame-sized (a binning half-extent over half the frame),
    off-screen (centre outside the frame), flipped (the normal turned to face the camera), ordinary"""
    pre = pre_cam(s, cam)
    box = cull_box(pre, s["alphas"])
    out = []
    for i in range(len(s["pws"])):
        pc, u, ext = pre["pc"][i], pre["u"][i], pre["ext"][i]
        cosang = abs(np.dot(pre["n"][i], pc)) / np.linalg.norm(pc)
        # screen-space lengths of the two axes at the centre (the projection's Jacobian)
        J = np.array([[cam["fx"] / pc[2], 0, -cam["fx"] * pc[0] / pc[2] ** 2],
                      [0, cam["fy"] / pc[2], -cam["fy"] * pc[1] / pc[2] ** 2]])
        ax = [np.linalg.norm(J @ (pre["scales"][i, j] * pre["axes"][i, :, j])) for j in (0, 1)]
        if not pre["keep"][i]:
            kind = "culled"
        elif s["alphas"][i] < 0.002:
            kind = "alpha-culled"
        elif (pre["areas"][i] == so.AREA_CAP).any():
            kind = "capped"
        elif np.isposinf(box[i]).any():
            kind = "unbounded"
        elif cosang < np.sin(np.deg2rad(3)):
            kind = "edge-on"
        elif cosang < np.sin(np.deg2rad(10)):
            kind = "grazing"
        elif max(ax) < 0.3:
            kind = "sub-pixel"
        elif max(ax) > 20 * min(ax):
            kind = "needle"
        elif ext.max() > max(W, H) / 2:
            kind = "frame-sized"
        elif not (0 <= u[0] < W and 0 <= u[1] < H):
            kind = "off-screen"
        elif pre["sgn"][i] < 0:
            kind = "flipped"
        else:
            kind = "ordinary"
        out.append(kind)
    return out


# camera -> the kind of special_scene's surfels 0-9 (built as: edge-on, grazing, sub-pixel, needle, frame-sized,
# off-screen, unbounded, alpha 0.0015, capped, flipped).  Each is another kind, or ordinary, in some other
# camera, but for the alpha-culled disk (its alpha is its own) and the needle (100:1, a needle wherever it
# is not culled); camera 1 culls every one.
SPECIAL_KINDS = [
    ["edge-on", "edge-on", "sub-pixel", "needle", "frame-sized", "off-screen", "unbounded", "alpha-culled", "capped",
     "flipped"],
    ["culled"] * 10,
    ["off-screen", "edge-on", "sub-pixel", "needle", "culled", "frame-sized", "culled", "alpha-culled", "culled",
     "frame-sized"],
    ["edge-on", "flipped", "sub-pixel", "needle", "culled", "ordinary", "frame-sized", "alpha-culled", "frame-sized",
     "flipped"],
    ["ordinary", "grazing", "sub-pixel", "needle", "frame-sized", "ordinary", "frame-sized", "alpha-culled", "needle",
     "flipped"],
    ["frame-sized", "grazing", "sub-pixel", "culled", "culled", "frame-sized", "culled", "alpha-culled", "culled",
     "frame-sized"],
    ["culled", "culled", "ordinary", "culled", "culled", "culled", "culled", "alpha-culled", "culled", "culled"],
]


def test_special_batch_degenerate_per_camera():
    W, H, cams, s = special_batch()
    got = [kinds_in(s, cam, W, H) for cam in cams]
    assert got == SPECIAL_KINDS, got
    for i in range(10):
        assert len({row[i] for row in got}) >= 2, i
    # the turned-away camera culls by depth: every centre behind it
    assert (pre_cam(s, cams[1])["pc"][:, 2] < 0).all()


# ---------------------------------------------------------------- frame boundaries
BOUNDARY = (3, 70, 45)  # C, W, H: 3 tile rows per frame, 3 pad rows and 10 pad columns


def boundary_batch(k=4):
    """-> (W, H, cams, scene, edge): C cameras well apart (0.05 rad, 0.15 m); for each camera c, 6 disks
    centred within 1.5 px of its frame's bottom edge (rows H - 1.5 to H + 0.5) and 6 on its first row
    (rows -0.5 to 1.5), 2-4 px across; 150 random disks.  edge[c] = (ids across camera c's bottom edge,
    ids on its first row)"""
    C, W, H = BOUNDARY
    rng = np.random.default_rng(45)
    cams = jittered_cameras(C, W, H, 0.8 * W, seed=70, ang=0.05, shift=0.15)
    parts, edge, n0 = [disks(rng, cams[0], W, H, 150, (2.0, 6.0)) + (rng.uniform(0.1, 0.9, 150),)], [], 150
    for c, cam in enumerate(cams):
        ids = []
        for v in ((H - 1.5, H + 0.5), (-0.5, 1.5)):
            pc, Rc, sc = disks(rng, cam, W, H, 6, (2.5, 4.0), sigma=(2.0, 4.0))
            x = np.linspace(6, W - 6, 6) + rng.uniform(-2, 2, 6)
            y = rng.uniform(*v, 6)
            pc[:, 0], pc[:, 1] = (x - cam["cx"]) * pc[:, 2] / cam["fx"], (y - cam["cy"]) * pc[:, 2] / cam["fy"]
            pws, rots = to_world(pc, Rc, cam)
            pc0 = pws @ cams[0]["Rcw"].astype(np.float64).T + cams[0]["tcw"]   # in camera 0's frame for build()
            parts.append((pc0, [cams[0]["Rcw"].astype(np.float64) @ so.quat_R(q[None])[0] for q in rots], sc,
                          rng.uniform(0.6, 0.9, 6)))
            ids.append(np.arange(n0, n0 + 6))
            n0 += 6
        edge.append(tuple(ids))
    return W, H, cams, build(rng, parts, cams[0], k), edge


def test_boundary_batch_reaches_both_edges():
    W, H, cams, s, edge = boundary_batch()
    gx, gy = (W + 15) // 16, (H + 15) // 16
    assert H % 16 and W % 16
    for c, cam in enumerate(cams):
        pre = pre_cam(s, cam)
        bins = so.bin_f32(H, W, pre)
        fwd = so.render(H, W, pre, s["alphas"], bins)
        bottom, top = edge[c]
        _, ranges, gsid, _ = bins
        tile_of = np.repeat(np.arange(gx * gy), ranges[:, 1] - ranges[:, 0])
        for ids, row in ((bottom, gy - 1), (top, 0)):
            for i in ids:
                assert np.isin(tile_of[gsid == i] // gx, [row]).any(), (c, i)
                assert abs(pre["u"][i, 1] - (H - 0.5 if row else 0.5)) <= 1.0
        # the bottom-edge disks are drawn on the frame's last row, the first-row ones on row 0
        for ids, r in ((bottom, H - 1), (top, 0)):
            xs = np.round(pre["u"][ids, 0]).astype(int)
            assert (fwd["alpha"][r, xs] > 0.1).all(), (c, r)
