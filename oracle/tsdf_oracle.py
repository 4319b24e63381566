"""fp64 model of TSDF fusion and marching-cubes extraction (DESIGN 3.17).  TEST INFRASTRUCTURE
ONLY -- imported by tests/ and benchmarks/, never by the product.

Grid: nx x ny x nz sample points, point g = (i, j, k) at origin + s (i, j, k); arrays are flat in
the order [nz, ny, nx] (x fastest), colour [3, N].  A new volume is tsdf 1, weight 0, colour 0.

integrate(): for every view in order, every point p: pc = Rcw p + tcw; skip unless pc.z > 0;
u = fx pc.x / pc.z + cx, v likewise; skip unless 0 <= u + 1/2 < W and 0 <= v + 1/2 < H; pixel
(x, y) = floor(u + 1/2, v + 1/2); D = depth[y, x]; skip unless D is finite and 0 < D <= depth_trunc;
sdf = D - pc.z; skip if sdf < -trunc; t = min(1, sdf / trunc);
T <- (T w + t) / (w + 1), C <- (C w + c[:, y, x]) / (w + 1), w <- w + 1.

extract(): observed = w > 0, inside = T < 0.  A cell (8 points, lowest corner g) is valid when all
8 corners are observed.  Edge (g, a) has a vertex when its ends differ in insideness and a valid
cell contains it, at p_g + s e_a f, f = T_g / (T_g - T_{g+e_a}), colour C_g + f (C_{g+e_a} - C_g);
vertices in order of (linear index of g, a).  Faces: valid cells in linear order, each cell's
triangles in table order (oracle/mc_table.py), as int indices into the vertices.
"""
import numpy as np

from . import mc_table

D64 = np.float64
CAM_ROW = 20  # ops.camera_table: Rcw (9, row-major), tcw (3), fx, fy, cx, cy, W, H, 2 unused


def new_volume(dims, color=True):
    nx, ny, nz = dims
    N = nx * ny * nz
    return {"tsdf": np.ones(N, D64), "weight": np.zeros(N, D64),
            "color": np.zeros((3, N), D64) if color else None}


def grid_index(dims):
    """(i, j, k) of every point, flat in [nz, ny, nx] order"""
    nx, ny, nz = dims
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    return np.stack([i.ravel(), j.ravel(), k.ravel()], axis=1)


def grid_points(dims, origin, voxel):
    return np.asarray(origin, D64) + D64(voxel) * grid_index(dims).astype(D64)


def integrate(vol, dims, origin, voxel, trunc, depth_trunc, cams, depth, color=None, margin=0.0):
    """Fuses views into `vol` (new_volume's dict, fp64) in place.  cams: [V, 20] camera table
    (ops.camera_table, as stored: fp32 values), depth [V, H, W], color [V, 3, H, W] or None.
    margin > 0: -> ambiguous[N], the points where some view makes a decision within a relative
    `margin` of its threshold (pc.z at 0, sdf at -trunc, D at depth_trunc, or u + 1/2 or v + 1/2
    at an integer when a candidate pixel fuses the point); a kernel's fp32 rounding may decide
    those the other way."""
    cams = np.asarray(cams, D64).reshape(-1, CAM_ROW)
    depth = np.asarray(depth, D64)
    V, H, W = depth.shape
    p = grid_points(dims, origin, voxel)
    amb = np.zeros(len(p), bool)
    for v in range(V):
        R, t = cams[v, :9].reshape(3, 3), cams[v, 9:12]
        fx, fy, cx, cy = cams[v, 12:16]
        pc = p @ R.T + t
        scale = np.abs(p) @ np.abs(R).T + np.abs(t)  # magnitude the fp32 pc is rounded against
        z = pc[:, 2]
        amb |= np.abs(z) <= margin * scale[:, 2]
        front = z > 0
        with np.errstate(divide="ignore", invalid="ignore"):
            u = fx * pc[:, 0] / z + cx
            vv = fy * pc[:, 1] / z + cy
            eu = margin * (np.abs(fx) * (scale[:, 0] + np.abs(pc[:, 0]) * scale[:, 2] / np.abs(z)) / np.abs(z)
                           + np.abs(cx) + np.abs(u) + 1)
            ev = margin * (np.abs(fy) * (scale[:, 1] + np.abs(pc[:, 1]) * scale[:, 2] / np.abs(z)) / np.abs(z)
                           + np.abs(cy) + np.abs(vv) + 1)
        hu, hv = u + 0.5, vv + 0.5
        with np.errstate(invalid="ignore"):
            inb = front & (hu >= 0) & (hu < W) & (hv >= 0) & (hv < H)
            near_u = front & (np.abs(hu - np.round(hu)) <= eu)
            near_v = front & (np.abs(hv - np.round(hv)) <= ev)

        def fuses(i, x, y):  # points i fused by pixel (x, y) of this view
            inside = (x >= 0) & (x < W) & (y >= 0) & (y < H)
            Dv = np.where(inside, depth[v, np.clip(y, 0, H - 1), np.clip(x, 0, W - 1)], np.nan)
            with np.errstate(invalid="ignore"):
                return inside & np.isfinite(Dv) & (Dv > 0) & (Dv <= depth_trunc) & (Dv - z[i] >= -trunc)

        # a pixel choice within the margin matters only when one of the candidate pixels fuses
        a = np.flatnonzero(near_u | near_v)
        if len(a):
            x0, y0 = np.floor(hu[a]), np.floor(hv[a])
            xs = [x0, np.where(near_u[a], 2 * np.round(hu[a]) - 1 - x0, x0)]
            ys = [y0, np.where(near_v[a], 2 * np.round(hv[a]) - 1 - y0, y0)]
            for xx in xs:
                for yy in ys:
                    amb[a] |= fuses(a, xx.astype(np.int64), yy.astype(np.int64))
        idx = np.flatnonzero(inb)
        x = np.floor(hu[idx]).astype(np.int64)
        y = np.floor(hv[idx]).astype(np.int64)
        D = depth[v, y, x]
        ok = np.isfinite(D) & (D > 0) & (D <= depth_trunc)
        with np.errstate(invalid="ignore"):
            sdf = D - z[idx]
            amb[idx] |= np.isfinite(D) & (D > 0) & (np.abs(D - depth_trunc) <= margin * np.abs(D))
            amb[idx] |= ok & (np.abs(sdf + trunc) <= margin * (np.abs(D) + scale[idx, 2] + trunc))
        ok &= sdf >= -trunc
        idx, x, y, sdf = idx[ok], x[ok], y[ok], sdf[ok]
        tv = np.minimum(1.0, sdf / trunc)
        w = vol["weight"][idx]
        vol["tsdf"][idx] = (vol["tsdf"][idx] * w + tv) / (w + 1)
        if vol["color"] is not None and color is not None:
            c = np.asarray(color[v], D64)[:, y, x]
            vol["color"][:, idx] = (vol["color"][:, idx] * w + c) / (w + 1)
        vol["weight"][idx] = w + 1
    return amb if margin > 0 else None


def _edge_offset(e):
    """the owner offset (dx, dy, dz) and the axis of cube edge e"""
    a, b, c, ob, oc = mc_table.edge_axes(e)
    o = [0, 0, 0]
    o[b], o[c] = ob, oc
    return o, a


def extract(dims, origin, voxel, tsdf, weight, color=None):
    """-> (verts[V, 3], faces[F, 3] int64, colors[V, 3] or None), fp64"""
    nx, ny, nz = dims
    T = np.asarray(tsdf, D64).reshape(nz, ny, nx)
    Wt = np.asarray(weight, D64).reshape(nz, ny, nx)
    Cg = None if color is None else np.asarray(color, D64).reshape(3, nz, ny, nx)
    table = mc_table.table()
    obs, ins = Wt > 0, T < 0
    cz, cy, cx = max(nz - 1, 0), max(ny - 1, 0), max(nx - 1, 0)
    cs = lambda a, d: a[d[2]:d[2] + cz, d[1]:d[1] + cy, d[0]:d[0] + cx]  # noqa: E731  corner d of every cell
    valid = np.ones((cz, cy, cx), bool)
    cls = np.zeros((cz, cy, cx), np.int64)
    for c in range(8):
        d = mc_table.corner_xyz(c)
        valid &= cs(obs, d)
        cls |= cs(ins, d).astype(np.int64) << c
    # edges of valid cells, by owner point and axis
    in_valid = np.zeros((3, nz, ny, nx), bool)
    for e in range(12):
        o, a = _edge_offset(e)
        in_valid[a, o[2]:o[2] + cz, o[1]:o[1] + cy, o[0]:o[0] + cx] |= valid
    cross = np.zeros((3, nz, ny, nx), bool)
    cross[0, :, :, :-1] = ins[:, :, :-1] != ins[:, :, 1:]
    cross[1, :, :-1, :] = ins[:, :-1, :] != ins[:, 1:, :]
    cross[2, :-1, :, :] = ins[:-1, :, :] != ins[1:, :, :]
    has = (in_valid & cross).reshape(3, -1).T  # [N, 3]: order (linear index, axis)
    ids = np.full(has.shape, -1, np.int64)
    ids[has] = np.arange(int(has.sum()))
    n_lin, ax = np.nonzero(has)
    g = grid_index(dims)[n_lin]
    step = np.array([1, nx, nx * ny])[ax]
    T0, T1 = T.ravel()[n_lin], T.ravel()[n_lin + step]
    f = T0 / (T0 - T1)
    verts = np.asarray(origin, D64) + D64(voxel) * g.astype(D64)
    verts[np.arange(len(ax)), ax] += D64(voxel) * f
    colors = None
    if Cg is not None:
        C = Cg.reshape(3, -1)
        colors = (C[:, n_lin] + f * (C[:, n_lin + step] - C[:, n_lin])).T
    # faces
    counts = np.array([len(t) for t in table])
    tri = np.zeros((256, mc_table.max_triangles(), 3), np.int64)
    for c in range(256):
        if table[c]:
            tri[c, :len(table[c])] = table[c]
    kk, jj, ii = np.nonzero(valid)
    cell_lin = (kk * ny + jj) * nx + ii
    ccls = cls[kk, jj, ii]
    rows = []
    for t in range(tri.shape[1]):
        sel = counts[ccls] > t
        if not sel.any():
            continue
        tv = np.empty((int(sel.sum()), 3), np.int64)
        for k in range(3):
            es = tri[ccls[sel], t, k]
            off = np.array([_edge_offset(e)[0] for e in range(12)])[es]
            axs = np.array([_edge_offset(e)[1] for e in range(12)])[es]
            own = ((kk[sel] + off[:, 2]) * ny + jj[sel] + off[:, 1]) * nx + ii[sel] + off[:, 0]
            tv[:, k] = ids[own, axs]
        rows.append((cell_lin[sel] * 8 + t, tv))
    if rows:
        key = np.concatenate([r[0] for r in rows])
        faces = np.concatenate([r[1] for r in rows])[np.argsort(key, kind="stable")]
    else:
        faces = np.zeros((0, 3), np.int64)
    assert (faces >= 0).all()
    return verts, faces, colors
