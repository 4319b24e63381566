"""Mesh extraction on the H100 (k_tsdf_integrate, k_tsdf_count / _ids / _emit, ops.tsdf_*,
mesh.TSDFVolume) against the fp64 model of oracle/tsdf_oracle.py, batched against one-view
launches, at a grid whose colour planes pass 2^31 elements, and end to end from surfel renders of a
sphere to a PLY mesh."""
import math

import numpy as np
import pytest
import torch
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from oracle import tsdf_oracle as tor

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = 2.0 ** -24  # fp32 unit roundoff
F32 = lambda x: float(np.float32(x))  # noqa: E731  the value the kernels are given


def _look_at(c, target=(0.0, 0.0, 0.0), up=(0.0, 0.0, 1.0)):
    """Rcw, tcw of a pinhole camera at c looking at target (camera z forward)"""
    c = np.asarray(c, np.float64)
    z = np.asarray(target, np.float64) - c
    z /= np.linalg.norm(z)
    x = np.cross(np.asarray(up, np.float64), z)
    if np.linalg.norm(x) < 1e-6:
        x = np.cross([0.0, 1.0, 0.0], z)
    x /= np.linalg.norm(x)
    R = np.stack([x, np.cross(z, x), z])
    return R, -R @ c


def _cameras(V, W, H, f, rng, radius=2.5, inside=False):
    from easygaussiansplatting_b200.gsfunction import Camera
    cams = []
    for v in range(V):
        if inside and v == 0:
            c, tgt = np.array([0.1, -0.05, 0.2]), np.array([0.8, 0.3, 0.1])
        else:
            d = rng.normal(size=3)
            c, tgt = radius * d / np.linalg.norm(d), rng.uniform(-0.2, 0.2, 3)
        R, t = _look_at(c, tgt)
        cams.append(Camera(W, H, f, f * 1.03, W / 2 - 0.3, H / 2 + 0.2, torch.tensor(R, dtype=torch.float32, device=DEV),
                           torch.tensor(t, dtype=torch.float32, device=DEV)))
    return cams


def _depth_maps(cams, W, H, rng, inside=False):
    """smooth surfaces at about the grid's centre, with holes: 0, negative, NaN, +-inf pixels"""
    V = len(cams)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    D = np.empty((V, H, W))
    for v in range(V):
        d0 = 0.9 if inside and v == 0 else 2.5 + rng.uniform(-0.3, 0.3)
        D[v] = d0 + 0.25 * np.sin(x * rng.uniform(0.01, 0.05) + rng.uniform(0, 6)) * np.cos(y * rng.uniform(0.01, 0.05))
    for bad in (0.0, -1.0, np.nan, np.inf, -np.inf):
        D.reshape(-1)[rng.choice(D.size, D.size // 50, replace=False)] = bad
    C = rng.uniform(0, 1, (V, 3, H, W))
    return D.astype(np.float32), C.astype(np.float32)


def _volume(dims, color):
    nx, ny, nz = dims
    tsdf = torch.ones((nz, ny, nx), dtype=torch.float32, device=DEV)
    weight = torch.zeros_like(tsdf)
    cg = torch.zeros((3, nz, ny, nx), dtype=torch.float32, device=DEV) if color else None
    return tsdf, weight, cg


CASES = [  # dims, origin, voxel, (W, H), f, V, colour, depth_trunc, a camera inside the grid
    ((37, 29, 41), (-0.9, -0.7, -1.0), 0.05, (203, 121), 150.0, 6, True, math.inf, False),
    ((37, 29, 41), (-0.9, -0.7, -1.0), 0.05, (203, 121), 150.0, 5, False, 2.6, True),
    ((96, 80, 64), (-1.2, -1.0, -0.8), 0.025, (640, 480), 420.0, 7, True, 2.7, True),
]


def _run_case(dims, origin, voxel, wh, f, V, color, depth_trunc, inside, seed=0):
    from easygaussiansplatting_b200 import ops
    rng = np.random.default_rng(seed)
    W, H = wh
    cams = _cameras(V, W, H, f, rng, inside=inside)
    D, Cimg = _depth_maps(cams, W, H, rng, inside=inside)
    table = ops.camera_table(cams)
    trunc = 5 * voxel
    tsdf, weight, cg = _volume(dims, color)
    Dt = torch.from_numpy(D).to(DEV)
    Ct = torch.from_numpy(Cimg).to(DEV) if color else None
    ops.tsdf_integrate(tsdf, weight, cg, origin, voxel, trunc, depth_trunc, table, Dt, Ct)
    torch.cuda.synchronize()
    return dict(cams=cams, table=table, D=D, C=Cimg, Dt=Dt, Ct=Ct, trunc=trunc, tsdf=tsdf, weight=weight, cg=cg)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_integration_matches_the_fp64_model(case):
    """Bound.  A view's t = min(1, (D - z) / trunc) from fp32 z = (Rcw p + tcw).z, with p itself
    rounded: |dz| <= 4 u S, S = |p| |Rcw| + |tcw| (per view, the row of z); D - z, 1 / trunc and
    the product round once each, so |dt| <= 4 u S / trunc + 3 u.  A unit-weight update
    (T w + t) (1 / (w + 1)) averages the errors it is given and adds three roundings of at most u
    (|T| <= 1), so after w updates |dT| <= 4 u S_max / trunc + (3 w + 3) u.  Colour, from exact
    inputs in [0, 1]: |dC| <= (3 w + 3) u.  Weights are counts: equal exactly.  Points where a view
    decides within 2^-21 (relative, four times the few ulps the projection rounds by) of a threshold
    are excluded and counted: they must stay under 1 % of the observed points."""
    dims, origin, voxel, wh, f, V, color, depth_trunc, inside = CASES[case]
    r = _run_case(*CASES[case])
    vol = tor.new_volume(dims, color)
    o32 = [F32(x) for x in origin]
    amb = tor.integrate(vol, dims, o32, F32(voxel), F32(r["trunc"]), F32(depth_trunc), r["table"].cpu().numpy(),
                        r["D"], r["C"] if color else None, margin=2.0 ** -21)
    ok = ~amb
    w = r["weight"].cpu().numpy().ravel()
    assert amb.sum() < 0.01 * (w > 0).sum(), amb.sum()
    assert (w[ok] == vol["weight"][ok]).all()
    assert (w > 0).sum() > 0.2 * w.size and w.max() >= 3
    p = tor.grid_points(dims, origin, voxel)
    R = r["table"].cpu().numpy()[:, :12].astype(np.float64)
    S = max((np.abs(p) @ np.abs(R[v, 6:9]) + abs(R[v, 11])).max() for v in range(V))
    tol = 4 * U * S / r["trunc"] + (3 * w + 3) * U
    got = r["tsdf"].cpu().numpy().ravel().astype(np.float64)
    err = np.abs(got - vol["tsdf"])[ok]
    assert (err <= tol[ok]).all(), (err.max(), np.argmax(err / tol[ok]))
    if color:
        cg = r["cg"].cpu().numpy().reshape(3, -1).astype(np.float64)
        cerr = np.abs(cg - vol["color"])[:, ok]
        assert (cerr <= (3 * w[ok] + 3) * U).all(), cerr.max()
    else:
        assert r["cg"] is None


def test_batched_views_are_bit_identical_to_one_view_launches():
    from easygaussiansplatting_b200 import ops
    dims, origin, voxel, wh, f, V, color, depth_trunc, inside = CASES[2]
    r = _run_case(*CASES[2])
    for chunks in ((1,) * V, (3, 4), (2, 2, 3)):
        tsdf, weight, cg = _volume(dims, True)
        v0 = 0
        for n in chunks:
            ops.tsdf_integrate(tsdf, weight, cg, origin, voxel, r["trunc"], depth_trunc, r["table"][v0:v0 + n],
                               r["Dt"][v0:v0 + n], r["Ct"][v0:v0 + n])
            v0 += n
        assert torch.equal(tsdf, r["tsdf"]) and torch.equal(weight, r["weight"]) and torch.equal(cg, r["cg"])
    # 70 views: more than one shared-memory chunk of cameras in one launch
    rng = np.random.default_rng(5)
    cams = _cameras(70, 64, 48, 60.0, rng)
    D, Cimg = _depth_maps(cams, 64, 48, rng)
    table = ops.camera_table(cams)
    Dt, Ct = torch.from_numpy(D).to(DEV), torch.from_numpy(Cimg).to(DEV)
    a, b = _volume((21, 19, 17), True), _volume((21, 19, 17), True)
    ops.tsdf_integrate(*a, (-1, -1, -1), 0.1, 0.3, math.inf, table, Dt, Ct)
    for v in range(70):
        ops.tsdf_integrate(*b, (-1, -1, -1), 0.1, 0.3, math.inf, table[v:v + 1], Dt[v:v + 1], Ct[v:v + 1])
    assert all(torch.equal(x, y) for x, y in zip(a, b)) and (a[1] > 40).any()


@pytest.mark.parametrize("case", [0, 2])
def test_extraction_matches_the_fp64_model_exactly(case):
    """On the kernel's own grid, insideness and validity are the same decisions in both, so counts,
    vertex order and faces are equal.  Positions: f = T0 / (T0 - T1) rounds twice (|df| <= 2 u,
    f in [0, 1]); p_g = fma(s, g, o) once and p_g + s f once more, so |dp| <= 2 u (|o| + s (n + 1)) +
    2 u s.  Colours: ca + f (cb - ca) in fp32: |dC| <= 4 u max|C|."""
    from easygaussiansplatting_b200 import ops
    dims, origin, voxel = CASES[case][:3]
    r = _run_case(*CASES[case])
    verts, faces, colors = ops.tsdf_extract(r["tsdf"], r["weight"], r["cg"], origin, voxel)
    tsdf = r["tsdf"].cpu().numpy().ravel()
    weight = r["weight"].cpu().numpy().ravel()
    cg = r["cg"].cpu().numpy().reshape(3, -1) if r["cg"] is not None else None
    v, fo, c = tor.extract(dims, [F32(x) for x in origin], F32(voxel), tsdf, weight, cg)
    assert len(fo) > 1000 and verts.shape == v.shape and faces.shape == fo.shape
    assert faces.dtype == torch.int32 and (faces.cpu().numpy() == fo).all()
    tol = 2 * U * (np.abs(origin).max() + voxel * (max(dims) + 1)) + 2 * U * voxel
    assert np.abs(verts.cpu().numpy() - v).max() <= tol
    if cg is not None:
        assert np.abs(colors.cpu().numpy() - c).max() <= 4 * U * max(1.0, np.abs(cg).max())
    else:
        assert colors is None


def test_ops_refuse_a_camera_table_of_another_size_and_emit_stays_in_its_buffers():
    import ctypes as C
    from easygaussiansplatting_b200 import _lib, ops
    dims, origin, voxel = CASES[0][:3]
    r = _run_case(*CASES[0])
    wrong = r["table"].clone()
    wrong[:, 16] += 1
    with pytest.raises(ValueError, match="width and height"):
        ops.tsdf_integrate(r["tsdf"], r["weight"], r["cg"], origin, voxel, r["trunc"], math.inf, wrong, r["Dt"],
                           r["Ct"])
    # an emit given smaller counts than its plan writes only inside them
    lib = _lib.load()
    nx, ny, nz = dims
    ws = torch.empty(lib.gsb_tsdf_extract_workspace_bytes(nx, ny, nz), dtype=torch.uint8, device=DEV)
    counts = (C.c_int64 * 2)()
    _lib.check(lib.gsb_tsdf_extract_plan(nx, ny, nz, r["tsdf"].data_ptr(), r["weight"].data_ptr(), ws.data_ptr(),
                                         ws.numel(), counts, None), lib)
    nv, nf = counts[0], counts[1]
    assert nv > 100 and nf > 100
    verts = torch.full((nv, 3), 7.0, device=DEV)
    faces = torch.full((nf, 3), -7, dtype=torch.int32, device=DEV)
    _lib.check(lib.gsb_tsdf_extract_emit(nx, ny, nz, *origin, voxel, r["tsdf"].data_ptr(), r["weight"].data_ptr(),
                                         None, ws.data_ptr(), ws.numel(), nv - 50, nf - 50, verts.data_ptr(), None,
                                         faces.data_ptr(), None), lib)
    torch.cuda.synchronize()
    ref_v, ref_f, _ = ops.tsdf_extract(r["tsdf"], r["weight"], None, origin, voxel)
    assert (verts[nv - 50:] == 7.0).all() and (faces[nf - 50:] == -7).all()
    assert torch.equal(verts[:nv - 50], ref_v[:nv - 50]) and torch.equal(faces[:nf - 50], ref_f[:nf - 50])


def test_empty_volumes_extract_to_empty_tensors():
    from easygaussiansplatting_b200 import ops
    for dims in ((40, 30, 20), (1, 30, 20), (40, 1, 20), (40, 30, 1)):
        tsdf, weight, cg = _volume(dims, True)
        if 1 in dims:  # observed, with a crossing, but no cells
            weight.fill_(1.0)
            tsdf[..., : dims[0] // 2] = -1.0
            tsdf[: dims[2] // 2] = -1.0
        v, f, c = ops.tsdf_extract(tsdf, weight, cg, (0, 0, 0), 0.1)
        assert v.shape == (0, 3) and f.shape == (0, 3) and c.shape == (0, 3) and v.is_cuda


def test_a_grid_past_2_31_colour_elements():
    """1024 x 1024 x 683 points (just over 2^31 / 3): colour plane 2 starts past 2^31 elements.
    One fronto-parallel view of constant depth and colour; the last planes are checked against
    the closed form t = min(1, (D - z) / trunc) and the view's colour."""
    from easygaussiansplatting_b200 import ops
    from easygaussiansplatting_b200.gsfunction import Camera
    dims = (1024, 1024, 683)
    assert dims[0] * dims[1] * dims[2] * 3 > 2 ** 31
    origin, voxel, trunc, D = (-5.12, -5.12, 0.5), 0.01, 0.05, 7.3
    try:
        tsdf, weight, cg = _volume(dims, True)
        cam = Camera(1024, 1024, 100.0, 100.0, 511.5, 511.5, torch.eye(3, device=DEV), torch.zeros(3, device=DEV))
        table = ops.camera_table([cam])
        depth = torch.full((1, 1024, 1024), D, device=DEV)
        color = torch.tensor([0.25, 0.5, 0.75], device=DEV).reshape(1, 3, 1, 1).expand(1, 3, 1024, 1024).contiguous()
        ops.tsdf_integrate(tsdf, weight, cg, origin, voxel, trunc, math.inf, table, depth, color)
        nz = dims[2]
        for k in (nz - 3, nz - 2, nz - 1):
            z = origin[2] + voxel * k
            sdf = D - z
            w = weight[k]
            exp_w = 1.0 if sdf >= -trunc else 0.0
            assert (w == exp_w).all(), k
            if exp_w:
                t = min(1.0, sdf / trunc)
                assert (tsdf[k] - t).abs().max().item() <= 4 * U * 8 / trunc + 6 * U
                for ch, val in enumerate((0.25, 0.5, 0.75)):
                    assert (cg[ch, k] == val).all(), (k, ch)
        assert (cg[2, : nz - 5] == 0.75 * (weight[: nz - 5] > 0)).all()
    finally:
        tsdf = weight = cg = None
        torch.cuda.empty_cache()


# ----------------------------------------------------------------------------- end to end

def _fibonacci(n):
    i = np.arange(n) + 0.5
    z = 1 - 2 * i / n
    phi = i * math.pi * (3 - math.sqrt(5))
    r = np.sqrt(1 - z * z)
    return np.stack([r * np.cos(phi), r * np.sin(phi), z], axis=1)


def _quat_from_normal(n):
    """(w, x, y, z) quaternions of frames whose third axis is n"""
    a = np.where(np.abs(n[:, 2:3]) < 0.9, [[0.0, 0.0, 1.0]], [[1.0, 0.0, 0.0]])
    t1 = np.cross(a, n)
    t1 /= np.linalg.norm(t1, axis=1, keepdims=True)
    t2 = np.cross(n, t1)
    R = np.stack([t1, t2, n], axis=2)  # columns
    w = np.sqrt(np.maximum(1 + R[:, 0, 0] + R[:, 1, 1] + R[:, 2, 2], 1e-12)) / 2
    x = (R[:, 2, 1] - R[:, 1, 2]) / (4 * w)
    y = (R[:, 0, 2] - R[:, 2, 0]) / (4 * w)
    z = (R[:, 1, 0] - R[:, 0, 1]) / (4 * w)
    return np.stack([w, x, y, z], axis=1)


def _sphere_renders(n=20000, n_cams=32):
    """-> (cameras, median depth where alpha >= 0.5 [V, H, W], images [V, 3, H, W]) of the surfel sphere"""
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionSurfelGeometry
    pw = _fibonacci(n)
    C0 = 0.28209479177387814
    rgb = np.where(pw[:, 2:3] > 0, [[1.0, 0.0, 0.0]], [[0.0, 0.0, 1.0]])
    T = lambda a: torch.tensor(np.asarray(a), dtype=torch.float32, device=DEV)  # noqa: E731
    pws, shs = T(pw), T((rgb - 0.5) / C0)
    scales, rots = T(np.full((n, 3), 0.02)), T(_quat_from_normal(pw))
    alphas = T(np.full((n, 1), 0.9))
    us = torch.zeros((n, 2), device=DEV)
    cams, depths, colors = [], [], []
    with torch.no_grad():
        for c in 3.0 * _fibonacci(n_cams):
            R, t = _look_at(c)
            cam = Camera(256, 256, 300.0, 300.0, 127.5, 127.5, T(R), T(t))
            image, depth, alpha, normal, dist, median, _ = GSFunctionSurfelGeometry.apply(
                pws, shs, alphas, scales, rots, us, cam)
            cams.append(cam)
            depths.append(torch.where(alpha >= 0.5, median, torch.zeros_like(median)))
            colors.append(image)
    return cams, torch.stack(depths), torch.stack(colors)


def _depth_points(cams, depths):
    """per view: camera centre c [3], ray directions per unit depth dw [H, W, 3] (world), depth D [H, W]"""
    out = []
    for cam, D in zip(cams, depths):
        R = cam.Rcw.cpu().numpy().astype(np.float64)
        t = cam.tcw.cpu().numpy().astype(np.float64)
        H, W = D.shape
        y, x = np.mgrid[0:H, 0:W].astype(np.float64)
        d = np.stack([(x - cam.cx) / cam.fx, (y - cam.cy) / cam.fy, np.ones_like(x)], -1)
        out.append((-R.T @ t, d @ R, D.cpu().numpy().astype(np.float64)))
    return out


def _exact_sphere_depth(cams):
    """the unit sphere's first-hit depth at every pixel centre (0 where the ray misses)"""
    out = []
    for c, dw, _ in _depth_points(cams, [torch.zeros(cam.height, cam.width) for cam in cams]):
        a, b, cc = (dw * dw).sum(-1), 2 * dw @ c, c @ c - 1
        disc = b * b - 4 * a * cc
        out.append(np.where(disc >= 0, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), 0.0))
    return np.array(out, np.float32)


def test_sphere_end_to_end_from_surfel_renders(tmp_path):
    """20k degree-0 surfels tangent to the unit sphere (sigma 0.02, alpha 0.9), red above the
    equator, blue below; 32 views at radius 3 (256 x 256, f = 300); median depth where alpha >= 0.5,
    fused into [-1.28, 1.28]^3 at voxel s = 0.02 with trunc = 5 s, extracted and written as PLY.
    Both bounds on the vertices' distance to the sphere are derived from the depth maps and the
    cameras, before the mesh is looked at.

    Per vertex.  A vertex lies on a grid edge (length s) between p_in (T < 0) and p_out (T >= 0),
    both observed.  The kernel reads the pixel whose centre is within 1/2 px of a point's projection
    on each axis, so at camera depth z the point is within l(z) = z / 2 sqrt(1/fx^2 + 1/fy^2) of
    the pixel-centre ray.  p_out has a view with D - z >= 0: it is within l of the segment from that
    camera to the depth sample X of the pixel, which enters the sphere by at most iota (the largest
    intrusion of such a segment over all pixels), so |v| >= 1 - iota - l - s.  p_in has a view with
    -trunc <= D - z < 0: it is within l of the pixel-centre ray between depths D and D + trunc,
    whose farthest point from the sphere is an end (|.| is convex along a line), at most omega
    outside (over all pixels), so |v| <= 1 + omega + l + s.  B_max = max(iota, omega) + l(z_max) + s,
    z_max the largest depth sample plus trunc.  omega includes the band behind depth samples on
    disks that overhang the silhouette (the projective TSDF's thickening); B_max must also stay
    within the ceiling trunc, which is asserted.

    On average.  With exact depth maps the fp64 model (oracle/tsdf_oracle.py) fuses and extracts a
    mesh at the same cameras, grid and truncation; its mean distance m_exact contains the
    projective TSDF's thickening behind silhouettes, the half-pixel lookup and the linear
    interpolation.  The surfel depth maps differ from the exact ones: a depth error e along a ray
    meeting the surface at incidence theta moves that view's zero by e cos theta, the radial
    distance r of the depth sample from the sphere, and the fused zero is an average of the views'
    zeros (weights 1 / cos theta), so it moves by at most the largest |r| of the views that see the
    point.  m_surfel = the mean over 20k points of the sphere of that largest |r| (first order), and
    the mean vertex distance is at most m_exact + m_surfel."""
    from easygaussiansplatting_b200 import ops
    from easygaussiansplatting_b200.gau_io import save_mesh_ply
    from easygaussiansplatting_b200.mesh import TSDFVolume
    from test_tsdf_cpu import read_mesh_ply

    s, trunc = 0.02, 0.1
    vol = TSDFVolume((-1.28,) * 3, (1.28,) * 3, s, trunc=trunc)
    assert vol.dims == (129, 129, 129)
    cams, depths, colors = _sphere_renders()
    for b in range(0, 32, 8):
        vol.integrate(depths[b:b + 8], cams[b:b + 8], colors[b:b + 8])
    # ---- the bounds, from the depth maps and cameras alone
    iota = omega = zmax = 0.0
    rows = _depth_points(cams, depths)
    for c, dw, D in rows:
        m = D > 0
        dw, D = dw[m], D[m]
        tc = np.clip(-(dw @ c) / (dw * dw).sum(-1), 0, D)  # closest approach of the camera -> sample segment
        iota = max(iota, (1 - np.linalg.norm(c + tc[:, None] * dw, axis=1)).max())
        far = np.maximum(np.linalg.norm(c + D[:, None] * dw, axis=1), np.linalg.norm(c + (D + trunc)[:, None] * dw, axis=1))
        omega = max(omega, (far - 1).max())
        zmax = max(zmax, D.max() + trunc)
    ell = zmax / 2 * math.sqrt(2) / 300.0
    b_max = max(iota, omega) + ell + s
    sph = _fibonacci(20000)
    worst = np.zeros(len(sph))
    for cam, (c, dw, D) in zip(cams, rows):
        R = cam.Rcw.cpu().numpy().astype(np.float64)
        t = cam.tcw.cpu().numpy().astype(np.float64)
        pc = sph @ R.T + t
        x = np.floor(cam.fx * pc[:, 0] / pc[:, 2] + cam.cx + 0.5).astype(int)
        y = np.floor(cam.fy * pc[:, 1] / pc[:, 2] + cam.cy + 0.5).astype(int)
        sees = ((sph * (c - sph)).sum(1) > 0) & (x >= 0) & (x < cam.width) & (y >= 0) & (y < cam.height)
        xs, ys = x[sees], y[sees]
        ok = D[ys, xs] > 0
        r = np.abs(np.linalg.norm(c + D[ys, xs, None] * dw[ys, xs], axis=1) - 1)
        idx = np.flatnonzero(sees)[ok]
        worst[idx] = np.maximum(worst[idx], r[ok])
    m_surfel = worst.mean()
    exact = tor.new_volume(vol.dims, color=False)
    tor.integrate(exact, vol.dims, [F32(x) for x in vol.origin], F32(s), F32(trunc), math.inf,
                  ops.camera_table(cams).cpu().numpy(), _exact_sphere_depth(cams))
    ve, _, _ = tor.extract(vol.dims, [F32(x) for x in vol.origin], F32(s), exact["tsdf"], exact["weight"])
    m_exact = np.abs(np.linalg.norm(ve, axis=1) - 1).mean()
    # ---- the mesh
    verts, faces, colors = vol.extract()
    v, f, c = verts.cpu().numpy().astype(np.float64), faces.cpu().numpy(), colors.cpu().numpy()
    # closed and consistently oriented: every directed edge once, its reverse once
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]).astype(np.int64)
    key = e[:, 0] * len(v) + e[:, 1]
    rkey = e[:, 1] * len(v) + e[:, 0]
    assert len(np.unique(key)) == len(key) and np.isin(rkey, key).all()
    # the largest component: chi = 2 and at least 99 % of the faces
    adj = coo_matrix((np.ones(len(e)), (e[:, 0], e[:, 1])), shape=(len(v), len(v)))
    ncomp, lab = connected_components(adj, directed=False)
    big = np.bincount(lab[f[:, 0]]).argmax()
    fb = f[lab[f[:, 0]] == big]
    assert len(fb) >= 0.99 * len(f)
    vb = np.unique(fb)
    assert len(vb) - 3 * len(fb) // 2 + len(fb) == 2
    dev = np.abs(np.linalg.norm(v, axis=1) - 1)
    print("sphere: max %.4f <= B_max %.4f (iota %.4f omega %.4f l %.4f); mean %.5f <= %.5f + %.5f"
          % (dev.max(), b_max, iota, omega, ell, dev.mean(), m_exact, m_surfel))
    assert b_max <= trunc and dev.max() <= b_max, (dev.max(), b_max)
    assert dev.mean() <= m_exact + m_surfel, (dev.mean(), m_exact, m_surfel)
    top, bot = v[:, 2] > 0.1, v[:, 2] < -0.1
    assert (c[top, 0] > c[top, 2]).all() and (c[bot, 2] > c[bot, 0]).all()
    save_mesh_ply(tmp_path / "sphere.ply", verts, faces, colors)
    v2, f2, c2 = read_mesh_ply(tmp_path / "sphere.ply")
    assert (v2 == verts.cpu().numpy()).all() and (f2 == f).all()
    assert (c2 == np.clip(np.rint(c.astype(np.float64) * 255), 0, 255)).all()
