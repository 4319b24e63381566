"""CPU checks of mesh extraction (DESIGN 3.17): the generated marching-cubes table for all 256
classes, the fp64 oracle's marching cubes on analytic SDFs and open surfaces, its integration
against closed forms, the C API's refusals, TSDFVolume's argument checks and the mesh PLY writer."""
import ctypes as C
import math
from collections import Counter

import numpy as np
import pytest

from oracle import mc_table as mc
from oracle import tsdf_oracle as tor


# ----------------------------------------------------------------------------- the table

def _directed_boundary(tris):
    """the directed edges of a triangle set that its reversed edges do not cancel"""
    e = Counter((t[i], t[(i + 1) % 3]) for t in tris for i in range(3))
    out = Counter()
    for (a, b), k in e.items():
        d = k - e.get((b, a), 0)
        if d > 0:
            out[(a, b)] = d
    return out


def test_table_boundary_is_the_face_rule_and_loops_close():
    for cls in range(256):
        tris = mc.triangles(cls)
        segs = mc.face_segments(cls)
        assert _directed_boundary(tris) == Counter(segs), cls
        ins = [(cls >> c) & 1 for c in range(8)]
        crossing = {e for e in range(12) if ins[mc.edge_corners(e)[0]] != ins[mc.edge_corners(e)[1]]}
        assert {p for p, _ in segs} == crossing and {q for _, q in segs} == crossing, cls
        assert sorted(e for lp in mc.loops(cls) for e in lp) == sorted(crossing), cls
        assert len(tris) == sum(len(lp) - 2 for lp in mc.loops(cls))
        assert all(len(set(t)) == 3 for t in tris)
    assert mc.triangles(0) == [] and mc.triangles(255) == []


def _face_pairing(cls, a, f):
    """the undirected segments of class cls on face (axis a, side f), as pairs of edge midpoints
    projected onto the face"""
    es = [x for x in mc.faces() if x[0][a] == 2 * f - 1][0][2]
    out = set()
    for p, q in mc.face_segments(cls):
        if p in es and q in es:
            mp = tuple(np.delete(mc.edge_mid(p), a)); mq = tuple(np.delete(mc.edge_mid(q), a))
            out.add(frozenset((mp, mq)))
    return out


def test_neighbouring_cells_cut_a_shared_face_alike():
    """the pairing on a face reads only the face's corners: the cell on either side agrees"""
    for a in range(3):
        for lo_cls in range(256):
            face_bits = [c for c in range(8) if mc.corner_xyz(c)[a] == 1]
            # the neighbour above along a has these corners on its side-0 face
            hi_cls = 0
            for c in face_bits:
                if (lo_cls >> c) & 1:
                    hi_cls |= 1 << (c & ~(1 << a))
            for other in (0, 0xff):  # any corners on the far face
                far = sum(1 << c for c in range(8) if mc.corner_xyz(c)[a] == 1)
                hc = hi_cls | (other & far)
                assert _face_pairing(lo_cls, a, 1) == _face_pairing(hc, a, 0), (a, lo_cls, hc)


def test_single_corner_normals_point_away_from_the_corner():
    for c in range(8):
        for cls, sign in ((1 << c, 1), (0xff ^ (1 << c), -1)):
            (t,) = mc.triangles(cls)
            P = [mc.edge_mid(e) for e in t]
            nrm = np.cross(P[1] - P[0], P[2] - P[0])
            assert sign * np.dot(nrm, np.mean(P, axis=0) - mc.corner_xyz(c)) > 0


def test_header_matches_the_generator():
    with open(mc.HEADER) as f:
        assert f.read() == mc.header_text()
    assert "#define MC_MAX_TRIS %d\n" % mc.max_triangles() in mc.header_text()
    assert mc.max_triangles() == 5


# ----------------------------------------------------------------------------- oracle marching cubes

def _topology(v, f):
    """-> (closed and consistently oriented, Euler characteristic, signed volume)"""
    e = Counter()
    for i in range(3):
        e.update(map(tuple, f[:, [i, (i + 1) % 3]]))
    ok = all(k == 1 and e.get((b, a), 0) == 1 for (a, b), k in e.items())
    n_edges = len({frozenset(x) for x in e})
    vol = np.einsum("ij,ij->i", v[f[:, 0]], np.cross(v[f[:, 1]], v[f[:, 2]])).sum() / 6
    return ok, len(v) - n_edges + len(f), vol


def _sphere(c, r):
    return (lambda p: np.linalg.norm(p - c, axis=-1) - r,
            lambda p: (p - c) / np.linalg.norm(p - c, axis=-1, keepdims=True))


def _torus(R, r):
    def sdf(p):
        q = np.sqrt(p[..., 0] ** 2 + p[..., 1] ** 2) - R
        return np.sqrt(q ** 2 + p[..., 2] ** 2) - r

    def grad(p):
        rho = np.sqrt(p[..., 0] ** 2 + p[..., 1] ** 2)
        c = np.stack([p[..., 0] / rho * R, p[..., 1] / rho * R, 0 * rho], axis=-1)
        d = p - c
        return d / np.linalg.norm(d, axis=-1, keepdims=True)
    return sdf, grad


def _union(A, B):
    return (lambda p: np.minimum(A[0](p), B[0](p)),
            lambda p: np.where((A[0](p) < B[0](p))[..., None], A[1](p), B[1](p)))


# name, (sdf, grad), chi, exact volume, exact area, largest curvature
SHAPES = [
    ("sphere", _sphere(np.zeros(3), 0.8), 2, 4 / 3 * math.pi * 0.8 ** 3, 4 * math.pi * 0.64, 1 / 0.8),
    ("torus", _torus(0.6, 0.25), 0, 2 * math.pi ** 2 * 0.6 * 0.25 ** 2, 4 * math.pi ** 2 * 0.6 * 0.25, 1 / 0.25),
    ("two spheres", _union(_sphere(np.array([0.5, 0, 0]), 0.35), _sphere(np.array([-0.5, 0, 0]), 0.35)), 4,
     2 * 4 / 3 * math.pi * 0.35 ** 3, 2 * 4 * math.pi * 0.35 ** 2, 1 / 0.35),
]


@pytest.mark.parametrize("name,shape,chi,vol,area,kappa", SHAPES, ids=[s[0] for s in SHAPES])
@pytest.mark.parametrize("n", [29, 41])
def test_oracle_marching_cubes_on_analytic_sdfs(name, shape, chi, vol, area, kappa, n):
    """Linear interpolation on an edge of length h puts a vertex within kappa h^2 / 2 of the zero
    set (the SDF's second derivative along a line is at most kappa near the surface), and a flat
    triangle of edges <= sqrt(3) h departs from the surface by at most kappa (sqrt(3) h)^2 / 8;
    the volume moves by at most the area times their sum, < area kappa h^2."""
    sdf, grad = shape
    h = 2.2 / (n - 1)
    origin = (-1.1, -1.1, -1.1)
    p = tor.grid_points((n, n, n), origin, h)
    v, f, _ = tor.extract((n, n, n), origin, h, sdf(p), np.ones(len(p)))
    ok, x, V = _topology(v, f)
    assert ok and x == chi
    assert V > 0 and abs(V - vol) < area * kappa * h * h
    assert np.abs(sdf(v)).max() <= kappa * h * h / 2
    cen = v[f].mean(axis=1)
    nrm = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    assert (np.einsum("ij,ij->i", nrm, grad(cen)) > 0).all()


def _boundary_vertices(f):
    e = Counter()
    for i in range(3):
        e.update(map(tuple, f[:, [i, (i + 1) % 3]]))
    return {x for (a, b) in e if (b, a) not in e for x in (a, b)}


def _vertex_edges(dims, tsdf, weight):
    """(owner point, axis) of every vertex, in the oracle's order"""
    v, f, _ = tor.extract(dims, (0, 0, 0), 1.0, tsdf, weight)
    g = np.floor(v).astype(int)  # voxel 1 at the origin: the owner point, and the axis that moved
    ax = np.argmax(v - g, axis=1)
    assert ((v - g > 0).sum(axis=1) == 1).all()  # no vertex sits on a grid point
    return v, f, g, ax


def _cells_of_edge(dims, g, a):
    """the lowest corners of the 4 cells around edge (g, a); None for a cell outside the grid"""
    b, c = [x for x in range(3) if x != a]
    out = []
    for ob in (0, 1):
        for oc in (0, 1):
            q = list(g)
            q[b] -= ob
            q[c] -= oc
            out.append(q if all(0 <= q[i] < dims[i] - 1 for i in range(3)) else None)
    return out


def _valid(dims, weight, q):
    nx, ny, nz = dims
    W = weight.reshape(nz, ny, nx)
    return all(W[q[2] + dz, q[1] + dy, q[0] + dx] > 0 for dx in (0, 1) for dy in (0, 1) for dz in (0, 1))


def test_open_surfaces_end_only_where_the_grid_or_the_observations_end():
    dims = (13, 11, 9)
    p = tor.grid_points(dims, (0, 0, 0), 1.0)
    # a tilted plane clipped by the grid: open edges only on boundary cells
    tsdf = p[:, 2] - 4.37 - 0.1 * p[:, 0] - 0.05 * p[:, 1]
    weight = np.ones(len(p))
    v, f, g, ax = _vertex_edges(dims, tsdf, weight)
    ok, _, _ = _topology(v, f)
    assert not ok
    bnd = _boundary_vertices(f)
    assert bnd
    for i in range(len(v)):
        on_edge = any(q is None for q in _cells_of_edge(dims, g[i], ax[i]))
        assert on_edge == (i in bnd), i
    # the same plane observed only for x < 7.5: open edges also where valid cells meet invalid ones
    weight = (p[:, 0] < 7.5).astype(float)
    v, f, g, ax = _vertex_edges(dims, tsdf, weight)
    bnd = _boundary_vertices(f)
    assert v[:, 0].max() <= 7 and len(bnd) > 0
    for i in range(len(v)):
        cells = _cells_of_edge(dims, g[i], ax[i])
        edge = any(q is None or not _valid(dims, weight, q) for q in cells)
        assert edge == (i in bnd), i


def test_extraction_of_empty_and_one_thick_grids():
    for dims in ((1, 5, 5), (5, 1, 5), (5, 5, 1), (1, 1, 1)):
        p = tor.grid_points(dims, (0, 0, 0), 1.0)
        v, f, c = tor.extract(dims, (0, 0, 0), 1.0, p[:, 0] - 2.5, np.ones(len(p)), np.ones((3, len(p))))
        assert v.shape == (0, 3) and f.shape == (0, 3) and c.shape == (0, 3)
    p = tor.grid_points((6, 6, 6), (0, 0, 0), 1.0)
    v, f, _ = tor.extract((6, 6, 6), (0, 0, 0), 1.0, p[:, 0] - 2.5, np.zeros(len(p)))
    assert len(v) == 0 and len(f) == 0


# ----------------------------------------------------------------------------- oracle integration

def _cam_row(R=np.eye(3), t=np.zeros(3), fx=100.0, fy=100.0, cx=15.5, cy=11.5, W=32, H=24):
    r = np.zeros(20)
    r[:9], r[9:12], r[12:18] = np.asarray(R).ravel(), t, (fx, fy, cx, cy, W, H)
    return r


def test_oracle_integration_against_closed_forms():
    """identity camera at the origin looking down +z, a fronto-parallel plane of depth D: a point
    at depth z in the image gets t = min(1, (D - z) / trunc) when D - z >= -trunc"""
    dims = (3, 3, 41)
    origin, s = (-0.06, -0.06, -1.0), 0.06   # x, y in {-0.06, 0, 0.06}, z from -1 to 1.4
    trunc, D = 0.05, 1.0
    p = tor.grid_points(dims, origin, s)
    z = p[:, 2]
    cam = _cam_row()[None]
    depth = np.full((1, 24, 32), D)
    color = np.zeros((1, 3, 24, 32)); color[0, 1] = 0.5
    vol = tor.new_volume(dims)
    tor.integrate(vol, dims, origin, s, trunc, math.inf, cam, depth, color)
    sdf = D - z
    with np.errstate(divide="ignore", invalid="ignore"):  # in the 32 x 24 image: 0 <= 100 x / z + 16 < 32, ...
        u, v = 100 * p[:, 0] / z + 16, 100 * p[:, 1] / z + 12
        seen = (z > 0) & (u >= 0) & (u < 32) & (v >= 0) & (v < 24)
    upd = seen & (sdf >= -trunc)
    assert upd.sum() > 40 and (vol["weight"] == upd).all()
    np.testing.assert_allclose(vol["tsdf"][upd], np.minimum(1, sdf[upd] / trunc), rtol=0, atol=1e-15)
    assert (vol["tsdf"][~upd] == 1).all() and (vol["color"][:, ~upd] == 0).all()
    assert (vol["color"][1, upd] == 0.5).all() and (vol["color"][0, upd] == 0).all()
    # a second view with another depth: the unit-weight average
    tor.integrate(vol, dims, origin, s, trunc, math.inf, cam, np.full((1, 24, 32), 0.7), np.ones((1, 3, 24, 32)))
    both = upd & (0.7 - z >= -trunc)
    np.testing.assert_allclose(vol["tsdf"][both], (np.minimum(1, sdf[both] / trunc) +
                                                   np.minimum(1, (0.7 - z[both]) / trunc)) / 2, atol=1e-15)
    assert (vol["weight"][both] == 2).all()
    np.testing.assert_allclose(vol["color"][1, both], 0.75)


@pytest.mark.parametrize("value", [0.0, -1.0, math.nan, math.inf, -math.inf])
def test_oracle_integration_skips_invalid_depth(value):
    dims = (4, 4, 4)
    vol = tor.new_volume(dims, color=False)
    tor.integrate(vol, dims, (-0.1, -0.1, 0.5), 0.05, 0.1, math.inf, _cam_row()[None], np.full((1, 24, 32), value))
    assert (vol["weight"] == 0).all() and (vol["tsdf"] == 1).all()


def test_oracle_integration_cuts_behind_camera_outside_image_and_truncations():
    dims = (40, 1, 30)
    origin, s = (-2.0, 0.0, -1.0), 0.1
    p = tor.grid_points(dims, origin, s)
    cam = _cam_row(fx=10.0, fy=10.0)  # W 32, H 24, cx 15.5: |x / z| <= 1.6 is in the image
    depth = np.full((1, 24, 32), 1.0)
    depth[:, :, :16] = 1.5  # left half deeper
    for depth_trunc in (math.inf, 1.2):
        vol = tor.new_volume(dims, color=False)
        tor.integrate(vol, dims, origin, s, 0.3, depth_trunc, cam[None], depth)
        z = p[:, 2]
        with np.errstate(divide="ignore", invalid="ignore"):
            u = 10 * p[:, 0] / z + 15.5
        inb = (z > 0) & (u + 0.5 >= 0) & (u + 0.5 < 32)
        D = np.where(u + 0.5 < 16, 1.5, 1.0)
        upd = inb & (D - z >= -0.3) & (D <= depth_trunc)
        assert (vol["weight"] == upd).all()
        assert (p[vol["weight"] > 0, 2] > 0).all()
    # a point just beyond -trunc is skipped, one at exactly -trunc is fused
    vol = tor.new_volume((1, 1, 2), color=False)
    tor.integrate(vol, (1, 1, 2), (0, 0, 1.25), 0.5, 0.25, math.inf, cam[None], depth)
    assert list(vol["weight"]) == [1, 0] and vol["tsdf"][0] == -1


def test_oracle_ambiguity_flags_half_pixel_points():
    dims = (1, 1, 1)
    cam = _cam_row(fx=10.0, cx=15.5, cy=11.3)
    vol = tor.new_volume(dims, color=False)
    # u + 1/2 = 10 * 0.05 / 1 + 15.5 + 0.5 = 16.5 is not at a pixel edge; 0.1 gives 17.0, which is
    amb = tor.integrate(vol, dims, (0.05, 0, 1), 0.1, 0.1, math.inf, cam[None], np.ones((1, 24, 32)), margin=1e-6)
    assert not amb[0]
    amb = tor.integrate(vol, dims, (0.1, 0, 1), 0.1, 0.1, math.inf, cam[None], np.ones((1, 24, 32)), margin=1e-6)
    assert amb[0]


# ----------------------------------------------------------------------------- host side

PTR = 0x10000000
INF, NAN = math.inf, math.nan


def _lib():
    from easygaussiansplatting_b200 import _lib as L, build
    build.build()
    return L.load()


def _integrate_args(**kw):
    a = dict(nx=8, ny=8, nz=8, ox=0.0, oy=0.0, oz=0.0, voxel=0.1, trunc=0.5, depth_trunc=INF, V=1, H=4, W=4,
             cams=PTR, depth=PTR, color=None, tsdf=PTR, weight=PTR, color_grid=None, stream=None)
    a.update(kw)
    return list(a.values())


INTEGRATE_REFUSALS = [
    ({"nx": 0}, "bad grid dimension"), ({"nz": -1}, "bad grid dimension"),
    ({"nx": 1 << 11, "ny": 1 << 10, "nz": 1 << 10}, "2^31 or more voxels"),
    ({"nx": 1291, "ny": 1291, "nz": 1291}, "2^31 or more voxels"),
    ({"voxel": 0.0}, "voxel must be"), ({"voxel": -1.0}, "voxel must be"), ({"voxel": NAN}, "voxel must be"),
    ({"voxel": INF}, "voxel must be"), ({"ox": NAN}, "origin not finite"),
    ({"trunc": 0.0}, "trunc must be"), ({"trunc": NAN}, "trunc must be"), ({"trunc": -0.1}, "trunc must be"),
    ({"depth_trunc": 0.0}, "depth_trunc must be"), ({"depth_trunc": NAN}, "depth_trunc must be"),
    ({"depth_trunc": -INF}, "depth_trunc must be"),
    ({"V": 0}, "V, H and W"), ({"H": 0}, "V, H and W"), ({"W": -3}, "V, H and W"),
    ({"color": PTR}, "one side only"), ({"color_grid": PTR}, "one side only"),
    ({"depth": None}, "null pointer"), ({"weight": None}, "null pointer"),
    ({"tsdf": PTR + 2}, "misaligned"),
]


@pytest.mark.parametrize("kw,text", INTEGRATE_REFUSALS, ids=[t + "-" + ",".join(k) for k, t in INTEGRATE_REFUSALS])
def test_tsdf_integrate_refusals(kw, text):
    lib = _lib()
    rc = lib.gsb_tsdf_integrate(*_integrate_args(**kw))
    assert rc == -1
    msg = lib.gsb_last_error().decode()
    assert msg.startswith("argument error: tsdf_integrate: ") and text in msg, msg


def test_tsdf_extract_refusals_and_workspace():
    lib = _lib()
    ws = lib.gsb_tsdf_extract_workspace_bytes
    assert ws(0, 4, 4) == 0 and ws(1 << 11, 1 << 10, 1 << 10) == 0
    assert ws(64, 64, 64) >= 12 * 64 ** 3 and ws(64, 64, 65) > ws(64, 64, 64)
    nb = ws(8, 8, 8)
    cnt = (C.c_int64 * 2)()

    def plan(**kw):
        a = dict(nx=8, ny=8, nz=8, tsdf=PTR, weight=PTR, ws=PTR, ws_bytes=nb, counts=cnt, stream=None)
        a.update(kw)
        rc = lib.gsb_tsdf_extract_plan(*a.values())
        return rc, lib.gsb_last_error().decode()

    def emit(**kw):
        a = dict(nx=8, ny=8, nz=8, ox=0.0, oy=0.0, oz=0.0, voxel=0.1, tsdf=PTR, weight=PTR, color_grid=None, ws=PTR,
                 ws_bytes=nb, V=10, F=10, verts=PTR, vcolors=None, faces=PTR, stream=None)
        a.update(kw)
        rc = lib.gsb_tsdf_extract_emit(*a.values())
        return rc, lib.gsb_last_error().decode()

    for kw, text in [({"ny": 0}, "bad grid dimension"), ({"nx": 1291, "ny": 1291, "nz": 1291}, "2^31 or more"),
                     ({"counts": None}, "counts_host is null"), ({"weight": None}, "null pointer"),
                     ({"ws": PTR + 16}, "misaligned"), ({"ws_bytes": nb - 1}, "workspace too small")]:
        rc, msg = plan(**kw)
        assert rc == -1 and "tsdf_extract_plan: " + text in msg, (kw, msg)
    for kw, text in [({"nz": 0}, "bad grid dimension"), ({"voxel": 0.0}, "voxel must be"),
                     ({"V": 1 << 31}, "vertex or face count out of range"), ({"F": 1 << 31}, "vertex or face count out of range"),
                     ({"V": -1}, "vertex or face count out of range"), ({"vcolors": PTR}, "vertex colours without a colour grid"),
                     ({"verts": None}, "null pointer"), ({"faces": None}, "null pointer"),
                     ({"ws_bytes": 0}, "workspace too small")]:
        rc, msg = emit(**kw)
        assert rc == -1 and "tsdf_extract_emit: " + text in msg, (kw, msg)
    # nothing to write: no launch, no error
    assert emit(V=0, F=0, verts=None, faces=None)[0] == 0


def test_tsdf_profile_ids():
    lib = _lib()
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    i = names.index("mcmc_noise")
    assert names[i + 1:i + 5] == ["tsdf_integrate", "tsdf_plan", "tsdf_emit", "surfel_forward"]


def test_tsdf_volume_argument_checks():
    torch = pytest.importorskip("torch")
    from easygaussiansplatting_b200.gsfunction import Camera
    from easygaussiansplatting_b200.mesh import TSDFVolume
    for kw in ({"lo": (0, 0)}, {"hi": (1, 1, 0)}, {"lo": (0, NAN, 0)}, {"voxel_size": 0}, {"voxel_size": NAN},
               {"trunc": 0}, {"trunc": INF}, {"depth_trunc": 0}, {"depth_trunc": NAN},
               {"voxel_size": 1e-3, "hi": (2, 2, 1)}):
        a = dict(lo=(0, 0, 0), hi=(1, 1, 1), voxel_size=0.1, device="cpu")
        a.update(kw)
        with pytest.raises(ValueError):
            TSDFVolume(**a)
    vol = TSDFVolume((-1, -1, -1), (1, 1, 1), 0.02, device="cpu")
    assert vol.dims == (101, 101, 101) and vol.trunc == pytest.approx(0.1)
    assert vol.tsdf.shape == (101, 101, 101) and vol.color.shape == (3, 101, 101, 101)
    assert (vol.tsdf == 1).all() and (vol.weight == 0).all() and (vol.color == 0).all()
    assert TSDFVolume((0, 0, 0), (1, 1, 1), 0.3, device="cpu", color=False).color is None
    assert TSDFVolume((0, 0, 0), (1, 1, 1), 0.3, device="cpu").dims == (5, 5, 5)
    R, t = torch.eye(3), torch.zeros(3)
    cam = Camera(8, 6, 10.0, 10.0, 3.5, 2.5, R, t)
    small = TSDFVolume((0, 0, 0), (1, 1, 1), 0.25, device="cpu")
    with pytest.raises(ValueError, match="8x6 but the depth map is 8x5"):
        small.integrate(torch.ones(5, 8), cam, torch.ones(3, 5, 8))
    with pytest.raises(ValueError, match="one camera"):
        small.integrate(torch.ones(2, 6, 8), [cam], torch.ones(2, 3, 6, 8))
    with pytest.raises(ValueError, match="one camera"):  # a lone camera with a batch of depth maps
        small.integrate(torch.ones(2, 6, 8), cam, torch.ones(2, 3, 6, 8))
    with pytest.raises(ValueError, match="needs colour"):
        small.integrate(torch.ones(6, 8), cam)
    fish = Camera(8, 6, 10.0, 10.0, 3.5, 2.5, R, t, camera_model="fisheye")
    with pytest.raises(ValueError, match="pinhole cameras only"):
        small.integrate(torch.ones(6, 8), fish, torch.ones(3, 6, 8))
    with pytest.raises(ValueError, match="has no colour"):
        TSDFVolume((0, 0, 0), (1, 1, 1), 0.25, device="cpu", color=False).integrate(torch.ones(6, 8), cam,
                                                                                    torch.ones(3, 6, 8))


def read_mesh_ply(path):
    """-> (verts, faces, colors or None) of save_mesh_ply's layout"""
    with open(path, "rb") as f:
        head = []
        while True:
            ln = f.readline().decode("ascii").strip()
            head.append(ln)
            if ln == "end_header":
                break
        nv = int([h for h in head if h.startswith("element vertex")][0].split()[-1])
        nf = int([h for h in head if h.startswith("element face")][0].split()[-1])
        rgb = "property uchar red" in head
        assert head[1] == "format binary_little_endian 1.0"
        assert "property list uchar int vertex_indices" in head
        vdt = [("xyz", "<f4", (3,))] + ([("rgb", "u1", (3,))] if rgb else [])
        v = np.frombuffer(f.read(nv * np.dtype(vdt).itemsize), vdt)
        fr = np.frombuffer(f.read(nf * 13), [("n", "u1"), ("idx", "<i4", (3,))])
        assert f.read() == b"" and (fr["n"] == 3).all()
    return v["xyz"].copy(), fr["idx"].copy(), (v["rgb"].copy() if rgb else None)


def test_save_mesh_ply_round_trip(tmp_path):
    from easygaussiansplatting_b200.gau_io import save_mesh_ply
    rng = np.random.default_rng(0)
    v = rng.normal(size=(17, 3)).astype(np.float32)
    f = rng.integers(0, 17, size=(23, 3)).astype(np.int32)
    c = rng.uniform(-0.1, 1.1, size=(17, 3)).astype(np.float32)
    save_mesh_ply(tmp_path / "a.ply", v, f, c)
    v2, f2, c2 = read_mesh_ply(tmp_path / "a.ply")
    assert (v2 == v).all() and (f2 == f).all()
    assert (c2 == np.clip(np.rint(c.astype(np.float64) * 255), 0, 255)).all()
    save_mesh_ply(tmp_path / "b.ply", v, f)
    v3, f3, c3 = read_mesh_ply(tmp_path / "b.ply")
    assert (v3 == v).all() and (f3 == f).all() and c3 is None
    save_mesh_ply(tmp_path / "c.ply", np.zeros((0, 3)), np.zeros((0, 3), int))
    assert read_mesh_ply(tmp_path / "c.ply")[0].shape == (0, 3)
    with pytest.raises(ValueError):
        save_mesh_ply(tmp_path / "d.ply", v, f + 17)
