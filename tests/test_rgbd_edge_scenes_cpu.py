"""The edge scenes of tests/test_gpu_rgbd_edges.py reach the edges they claim, checked with the fp64
RGB-D oracle alone (no GPU): patch counts and survivor blocks of the boundary scene, the
contrib of its opaque stacks, the early-termination fraction of the dense scene, the opacity
clamp and the never-composited tiny opacities, the coverage of the huge and needle scene, and
the dead tiles and 64-bit sort keys of the 4K scene.  The GPU tests assert the same claims on the
device's own inputs; this file makes a scene edit that loses its edge fail before any GPU run."""
import numpy as np

from oracle import oracle as orc
from oracle import rgbd_oracle as orgbd
from test_gpu_parity import (DEAD_H, DEAD_W, boundary_frame, boundary_scene, clamp_scene, dead_sparse_scene,
                             dense_scene, huge_needle_scene)
from test_gpu_rgbd_edges import boundary_claims, dead_sparse_claims, dense_claims

f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)


def part_inputs(parts):
    """gaussians_in_tile groups -> the splat inputs (us, cinv2ds, alphas, depths, colors, areas)"""
    cols = [np.concatenate([p[i] for p in parts]) for i in range(6)]
    return f32(cols[0]), f32(cols[1]), f32(cols[2]), f32(cols[3]), f32(cols[4]), np.ascontiguousarray(cols[5])


def scene_inputs(sc):
    """a synthetic scene through the oracle's five stages -> the splat inputs"""
    W, H = sc["width"], sc["height"]
    us, pcs, depths, _ = orc.project(sc["pws"], sc["Rcw"], sc["tcw"], sc["fx"], sc["fy"], sc["cx"], sc["cy"])
    d32 = f32(depths)
    c3 = orc.compute_cov3d(sc["rots"], sc["scales"], d32)[0]
    c2 = orc.compute_cov2d(f32(c3), f32(pcs), sc["Rcw"], d32, sc["fx"], sc["fy"], W, H)[0]
    col = orc.sh2color(sc["shs"], sc["pws"], sc["twc"])[0]
    ci, areas, _ = orc.inverse_cov2d(f32(c2), d32)
    return f32(us), f32(ci), f32(sc["alphas"]), d32, f32(col), areas


def render(H, W, inputs):
    us, ci, al, d, col, ar = inputs
    return orgbd.splat_rgbd(H, W, us, ci, al, d.copy(), col, ar.copy())


def test_boundary_scene_reaches_its_edges():
    """(with the per-tile depth offsets of the RGB-D case: the edges do not depend on depth)"""
    for z0s in (None, np.random.default_rng(70).uniform(1.0, 20.0, 64)):
        parts, expect, survivor_tiles, stack_tiles = boundary_scene(np.random.default_rng(7), z0s=z0s)
        W, H = boundary_frame(expect)
        ref = render(H, W, part_inputs(parts))
        boundary_claims(ref, expect, survivor_tiles, stack_tiles)
        assert set(survivor_tiles.values()) == {6, 7, 8, 9, 16, 17}
        assert sorted(stack_tiles.values()) == [32, 33, 34]
        if z0s is not None:   # list order inside a tile is still the build order
            lens = ref["ranges"][:, 1] - ref["ranges"][:, 0]
            for i in expect:
                ids = ref["gsid"][ref["ranges"][i, 0]:ref["ranges"][i, 1]]
                assert np.array_equal(ids, np.sort(ids)) and len(ids) == lens[i]


def test_dense_scene_terminates_early():
    sc = dense_scene()
    ref = render(sc["height"], sc["width"], scene_inputs(sc))
    dense_claims(ref)


def test_clamp_scene_reaches_the_clamp_and_tiny_alphas_never_composite():
    sc = clamp_scene()
    W, H = sc["width"], sc["height"]
    inputs = scene_inputs(sc)
    us, ci, al, d, col, ar = inputs
    ref = render(H, W, inputs)
    # an opacity-1.0 Gaussian whose nearest pixel has g >= 0.99: alpha' is clamped there
    full = np.flatnonzero((al == 1.0) & (d > 0))
    px = np.rint(us[full]).astype(np.int64)
    inside = (px[:, 0] >= 0) & (px[:, 0] < W) & (px[:, 1] >= 0) & (px[:, 1] < H)
    dx, dy = (px - us[full].astype(np.float64)).T
    c = ci[full].astype(np.float64)
    g = np.exp(-0.5 * (c[:, 0] * dx * dx + c[:, 2] * dy * dy) - c[:, 1] * dx * dy)
    assert (inside & (g >= 0.99)).sum() >= 3
    # alpha 0.001 can never reach the 0.002 skip threshold: no gradient at all
    rng = np.random.default_rng(2)
    dl = rng.normal(size=(3, H, W))
    dld, dla = rng.normal(size=(H, W)), rng.normal(size=(H, W))
    du, dc, da, dcol, dz = orgbd.splat_backward_rgbd(H, W, us, ci, al, col, ref["z"], ref, dl, dld, dla)
    tiny = al == np.float32(0.001)
    assert tiny.sum() > 40 and (al == np.float32(0.002)).sum() > 20
    for x in (du, dc, da, dcol, dz):
        assert not x.reshape(len(al), -1)[tiny].any()
    assert np.abs(dz).max() > 0


def test_huge_needle_scene_covers_every_tile():
    sc = huge_needle_scene()
    N = len(sc["pws"])
    ref = render(sc["height"], sc["width"], scene_inputs(sc))
    lens = ref["ranges"][:, 1] - ref["ranges"][:, 0]
    assert ref["P"] > 15 * N and lens.min() > 30


def test_dead_sparse_scene_has_dead_tiles_and_64bit_keys():
    parts = dead_sparse_scene(np.random.default_rng(11))
    ref = render(DEAD_H, DEAD_W, part_inputs(parts))
    dead = dead_sparse_claims(ref)
    assert dead.sum() == dead.size // 2
    dead_px = np.repeat(np.repeat(dead, 16, axis=0), 16, axis=1)
    assert not ref["depth"][dead_px].any() and not ref["alpha"][dead_px].any()
    assert ref["z"][ref["gsid"]].max() > 900.0
