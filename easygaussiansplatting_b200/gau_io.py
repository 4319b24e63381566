"""Gaussian scene I/O on the C ABI (SURVEY 8f row N3): the mirror of gsplat/gau_io.py
(reference :7-12 gsdata_type, :60-107 load_ply, :128-153 load_gs / save_gs /
save_training_params, :156-183 get_example_gs, :15-57/:110-126 rotate_gaussian) and of
gsmodel.get_training_params (gsmodel.py:95-129).

The host only parses the PLY header and moves bytes; the per-value work (sigmoid / exp /
normalise, the f_rest channel-major -> coefficient-major transpose, the logit / log inverse
and the SH padding) runs on the GPU, so a checkpoint goes disk -> pinned host -> HBM ->
training tensors without a float ever being touched by numpy:

    params, adam_groups = load_training_params("point_cloud.ply")     # device tensors
    gs = load_ply("point_cloud.ply")                                  # the reference's recarray

No `plyfile` dependency.  Only binary_little_endian PLY whose vertex properties are all
float32 is accepted -- the layout official 3DGS checkpoints use and the only one the
reference's column arithmetic (sh_dim = n_properties - 14, :82) is meaningful for.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import GAUSSIAN_TENSORS, GAUSSIAN_WIDTHS
from .density import _check, _ptr, _stream, gaussians_struct

_FLOAT_NAMES = ("float", "float32")


def gsdata_type(sh_dim):
    """gau_io.py:7-12"""
    return [("pw", "<f4", (3,)), ("rot", "<f4", (4,)), ("scale", "<f4", (3,)), ("alpha", "<f4"),
            ("sh", "<f4", (sh_dim,))]


# ----------------------------------------------------------------------------- PLY header

def read_ply_header(f):
    """-> (vertex count, property names, byte offset of the vertex block)"""
    if f.readline().strip() != b"ply":
        raise ValueError("not a PLY file")
    fmt, count, names, in_vertex, seen_vertex = None, 0, [], False, False
    while True:
        line = f.readline()
        if not line:
            raise ValueError("PLY header is not terminated")
        tok = line.decode("ascii").split()
        if not tok or tok[0] == "comment":
            continue
        if tok[0] == "end_header":
            break
        if tok[0] == "format":
            fmt = tok[1]
        elif tok[0] == "element":
            in_vertex = tok[1] == "vertex"
            if in_vertex:
                if seen_vertex:
                    raise ValueError("two vertex elements")
                seen_vertex, count = True, int(tok[2])
            elif not seen_vertex:
                raise ValueError("the vertex element must come first")
        elif tok[0] == "property" and in_vertex:
            if tok[1] not in _FLOAT_NAMES:
                raise ValueError("vertex property %r is %s; only float32 columns are supported" % (tok[-1], tok[1]))
            names.append(tok[2])
    if fmt != "binary_little_endian":
        raise ValueError("only binary_little_endian PLY is supported, got %r" % fmt)
    return count, names, f.tell()


def ply_column_map(names):
    """source column of each gs-row column (pw3 rot4 scale3 alpha sh[sh_dim]); f_rest_* is
    stored channel-major [3, k] and the reference re-orders it to [k, 3] (gau_io.py:91)"""
    col = {nm: i for i, nm in enumerate(names)}
    sh_dim = len(names) - 14                                 # gau_io.py:82
    if sh_dim not in (3, 12, 27, 48):
        raise ValueError("PLY has %d properties: sh_dim = %d is not 3, 12, 27 or 48" % (len(names), sh_dim))
    try:
        cmap = [col["x"], col["y"], col["z"]] + [col["rot_%d" % i] for i in range(4)] + \
            [col["scale_%d" % i] for i in range(3)] + [col["opacity"]] + [col["f_dc_%d" % i] for i in range(3)]
        k = (sh_dim - 3) // 3
        for j in range(sh_dim - 3):                          # output (coef j // 3, channel j % 3)
            cmap.append(col["f_rest_%d" % ((j % 3) * k + j // 3)])
    except KeyError as e:
        raise ValueError("PLY is missing property %s" % e)
    return np.asarray(cmap, np.int32), sh_dim


# ----------------------------------------------------------------------------- device paths

def ply_to_gs_rows(path, device="cuda"):
    """disk -> device gs rows [N, 11 + sh_dim] (activated values, the .npy record layout)"""
    lib = _lib.load()
    with open(path, "rb") as f:
        count, names, off = read_ply_header(f)
        cmap, sh_dim = ply_column_map(names)
        stride = len(names)
        host = torch.empty((count, stride), dtype=torch.float32, pin_memory=torch.cuda.is_available())
        buf = host.numpy().reshape(-1).view(np.uint8)
        got = f.readinto(memoryview(buf))
        if got != count * stride * 4:
            raise ValueError("PLY vertex block is truncated: %d of %d bytes" % (got, count * stride * 4))
    if not torch.cuda.is_available():
        raise RuntimeError("gau_io needs a CUDA device: the record arithmetic runs on the GPU (no CPU fallback)")
    rows = host.to(device, non_blocking=True)
    dmap = torch.from_numpy(cmap).to(device)
    out = torch.empty((count, 11 + sh_dim), dtype=torch.float32, device=device)
    _lib.check(lib.gsb_ply_rows_to_gs(count, stride, sh_dim, _ptr(rows), _ptr(dmap), _ptr(out), _stream()), lib)
    return out, sh_dim


def gs_rows_to_params(rows, sh_dim):
    """get_training_params' arithmetic (gsmodel.py:95-113) on device gs rows -> dict of the six
    raw training tensors (leaves with requires_grad, like the reference's)"""
    lib = _lib.load()
    N = rows.shape[0]
    rows = _check(rows, "gs rows", (N, 11 + sh_dim))
    out = {k: torch.empty((N, w), dtype=torch.float32, device=rows.device)
           for k, w in zip(GAUSSIAN_TENSORS, GAUSSIAN_WIDTHS)}
    g, keep = gaussians_struct(out)
    _lib.check(lib.gsb_gs_to_params(N, sh_dim, _ptr(rows), C.byref(g), _stream()), lib)
    return {k: t.requires_grad_() for k, t in out.items()}


def params_to_gs_rows(training_params):
    """save_training_params' arithmetic (gau_io.py:138-148) -> device gs rows [N, 59]"""
    lib = _lib.load()
    N = training_params["pws"].shape[0]
    src = {k: _check(training_params[k].detach(), "training_params[%r]" % k, (N, w))
           for k, w in zip(GAUSSIAN_TENSORS, GAUSSIAN_WIDTHS)}
    rows = torch.empty((N, 59), dtype=torch.float32, device=src["pws"].device)
    g, keep = gaussians_struct(src)
    _lib.check(lib.gsb_params_to_gs(N, C.byref(g), _ptr(rows), _stream()), lib)
    return rows


def bake_filter3d(training_params, filter3d):
    """The plain 3DGS parameters of a model trained with the Mip-Splatting 3D filter: the six raw
    training tensors whose activated scales and opacities are the filtered s' = sqrt(s^2 + f^2) and
    alpha' = alpha prod s / s' (ops.filter3d_apply), so a renderer, viewer or PLY consumer that
    knows nothing of the filter draws the filtered model.  Bake before saving.
    -> dict of the six raw tensors (new leaves with requires_grad, as gs_rows_to_params)."""
    from . import ops
    rows = params_to_gs_rows(training_params)  # activated: pw 3 | rot 4 | scale 3 | alpha 1 | sh 48
    sf, af = ops.filter3d_apply(rows[:, 7:10], rows[:, 10], filter3d)
    rows[:, 7:10] = sf
    rows[:, 10] = af
    return gs_rows_to_params(rows, 48)


def _rows_to_recarray(rows, sh_dim):
    host = rows.cpu().numpy()
    return np.rec.array(np.ascontiguousarray(host).view(np.dtype(gsdata_type(sh_dim))).reshape(-1))


def _recarray_to_rows(gs, device="cuda"):
    sh = np.asarray(gs["sh"])
    sh_dim = sh.shape[1] if sh.ndim == 2 else 1
    want = np.dtype(gsdata_type(sh_dim))
    arr = np.ascontiguousarray(np.asarray(gs).astype(want, copy=False))
    flat = arr.view("<f4").reshape(len(arr), 11 + sh_dim)
    return torch.from_numpy(flat).to(device), sh_dim


ADAM_LRS = (("pws", 0.001), ("low_shs", 0.001), ("high_shs", 0.001 / 20), ("alphas_raw", 0.05),
            ("scales_raw", 0.005), ("rots_raw", 0.001))


def adam_groups(params):
    """the optimizer groups of get_training_params (gsmodel.py:118-127)"""
    return [{"params": [params[k]], "lr": lr, "name": k} for k, lr in ADAM_LRS]


# ----------------------------------------------------------------------------- reference surface

def load_ply(path, T=None):
    """gau_io.py:60-107 -> np.recarray with dtype gsdata_type(sh_dim)"""
    rows, sh_dim = ply_to_gs_rows(path)
    return _rows_to_recarray(rows, sh_dim)


def load_gs(fn):
    """gau_io.py:128-135 (raises instead of exit(0) on an unknown suffix)"""
    if fn.endswith(".ply"):
        return load_ply(fn)
    if fn.endswith(".npy"):
        return np.load(fn)
    raise ValueError("%s is not a supported file." % fn)


def save_gs(fn, gs):
    """gau_io.py:137-138"""
    np.save(fn, gs)


def get_training_params(gs):
    """gsmodel.py:95-129: recarray -> (params dict of CUDA leaves, Adam param groups)"""
    rows, sh_dim = _recarray_to_rows(gs)
    params = gs_rows_to_params(rows, sh_dim)
    return params, adam_groups(params)


def load_training_params(path):
    """disk -> training tensors without leaving the device (load_gs + get_training_params)"""
    if path.endswith(".ply"):
        rows, sh_dim = ply_to_gs_rows(path)
    else:
        rows, sh_dim = _recarray_to_rows(load_gs(path))
    params = gs_rows_to_params(rows, sh_dim)
    return params, adam_groups(params)


def save_training_params(fn, training_params):
    """gau_io.py:138-153: activated values as a .npy structured array with sh_dim = 48"""
    np.save(fn, _rows_to_recarray(params_to_gs_rows(training_params), 48))


def save_ply(path, gs):
    """inverse of load_ply (no reference counterpart): writes the official 3DGS layout so a
    scene trained here opens in the stock viewers.  Host-side, not a hot path."""
    gs = np.asarray(gs)
    sh = np.asarray(gs["sh"], np.float32)
    N, sh_dim = sh.shape
    k = (sh_dim - 3) // 3
    rest = sh[:, 3:].reshape(N, k, 3).transpose(0, 2, 1).reshape(N, sh_dim - 3)
    a = np.asarray(gs["alpha"], np.float64)
    names = ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] + \
        ["f_rest_%d" % i for i in range(sh_dim - 3)] + ["opacity", "scale_0", "scale_1", "scale_2",
                                                        "rot_0", "rot_1", "rot_2", "rot_3"]
    rows = np.concatenate([gs["pw"], np.zeros((N, 3)), sh[:, :3], rest, np.log(a / (1 - a))[:, None],
                           np.log(np.asarray(gs["scale"], np.float64)), gs["rot"]], axis=1)
    with open(path, "wb") as f:
        f.write(("ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % N).encode("ascii"))
        f.write("".join("property float %s\n" % s for s in names).encode("ascii"))
        f.write(b"end_header\n")
        f.write(np.ascontiguousarray(rows, "<f4").tobytes())


def save_compressed(path, training_params, sh_clusters=65536, iters=10, generator=None):
    """Writes the six raw training tensors as one compressed scene file (compress.py, DESIGN 3.24):
    the SH rows vector-quantised against a k-means codebook of min(sh_clusters, N) rows (`iters`
    Lloyd iterations, initial centroids drawn with `generator`), the other attributes as 8 / 16-bit
    codes, in an np.savez_compressed archive written to `path` as given.  19 N + 45 K bytes of codes
    before deflate, against 248 N for save_ply.
    A model trained with the Mip-Splatting 3D filter is baked first (bake_filter3d): the file holds
    plain 3DGS parameters.  Raises ValueError on N = 0 or non-finite parameters."""
    from . import compress as cz
    for k in GAUSSIAN_TENSORS:
        if k not in training_params:
            raise ValueError("training_params has no %r" % k)
    N = training_params["pws"].shape[0]
    if N == 0:
        raise ValueError("there is nothing to save (N = 0)")
    for k in GAUSSIAN_TENSORS:
        if not bool(torch.isfinite(training_params[k].detach()).all()):
            raise ValueError("training_params[%r] is not finite" % k)
    cz.write_npz(path, cz.to_numpy(cz.compress(training_params, sh_clusters, iters, generator)))


def load_compressed(path, device="cuda"):
    """save_compressed's file -> (params, adam_groups) as load_training_params returns them: the six
    decoded raw tensors on `device`, leaves with requires_grad.  Reads without pickles; raises
    ValueError on an unknown format or version, a missing array, a wrong dtype or shape, N or K that
    disagree between the arrays, or a label >= K."""
    from . import compress as cz
    arrays, _ = cz.read_npz(path)
    params = cz.decompress(cz.to_device(arrays, device))
    params = {k: t.requires_grad_() for k, t in params.items()}
    return params, adam_groups(params)


def save_mesh_ply(path, verts, faces, colors=None):
    """Writes a triangle mesh (mesh.TSDFVolume.extract's output; tensors or arrays) as binary
    little-endian PLY: float x, y, z, with colors[V, 3] in [0, 1] also uchar red, green, blue
    (round(255 c), clamped), and a `uchar int vertex_indices` face list."""
    as_np = lambda a: a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)  # noqa: E731
    v = as_np(verts).astype("<f4").reshape(-1, 3)
    fc = as_np(faces).astype("<i4").reshape(-1, 3)
    if len(fc) and (fc.min() < 0 or fc.max() >= len(v)):
        raise ValueError("faces index outside the %d vertices" % len(v))
    vdt = [("xyz", "<f4", (3,))]
    if colors is not None:
        c = as_np(colors).reshape(-1, 3)
        if len(c) != len(v):
            raise ValueError("colors must have one row per vertex")
        vdt.append(("rgb", "u1", (3,)))
    vrows = np.empty(len(v), vdt)
    vrows["xyz"] = v
    if colors is not None:
        vrows["rgb"] = np.clip(np.rint(c.astype(np.float64) * 255), 0, 255).astype(np.uint8)
    frows = np.empty(len(fc), [("n", "u1"), ("idx", "<i4", (3,))])
    frows["n"], frows["idx"] = 3, fc
    head = "ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % len(v)
    head += "property float x\nproperty float y\nproperty float z\n"
    if colors is not None:
        head += "property uchar red\nproperty uchar green\nproperty uchar blue\n"
    head += "element face %d\nproperty list uchar int vertex_indices\nend_header\n" % len(fc)
    with open(path, "wb") as f:
        f.write(head.encode("ascii"))
        f.write(vrows.tobytes())
        f.write(frows.tobytes())


def get_example_gs():
    """gau_io.py:156-183: the 4-Gaussian test scene"""
    s = 1.772484
    gs = np.zeros(4, dtype=gsdata_type(3))
    gs["pw"] = [[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]]
    gs["rot"] = [[1, 0, 0, 0]] * 4
    gs["scale"] = [[0.05, 0.05, 0.05], [0.2, 0.05, 0.05], [0.05, 0.2, 0.05], [0.05, 0.05, 0.2]]
    gs["alpha"] = 1.0
    gs["sh"] = [[s, -s, s], [s, -s, -s], [-s, s, -s], [-s, -s, s]]
    return gs


def matrix_to_quaternion(matrices):
    """gau_io.py:15-57: rotation matrices [N,3,3] -> (w,x,y,z), the usual four-branch form"""
    m = np.asarray(matrices, np.float64)
    tr = 1 + m[:, 0, 0] + m[:, 1, 1] + m[:, 2, 2]
    q = np.ones((m.shape[0], 4))
    d = np.stack([m[:, 0, 0], m[:, 1, 1], m[:, 2, 2]], axis=1)
    pos = tr > 1e-7
    branch = np.where(pos, 3, np.where((d[:, 0] > d[:, 1]) & (d[:, 0] > d[:, 2]), 0, np.where(d[:, 1] > d[:, 2], 1, 2)))
    with np.errstate(invalid="ignore", divide="ignore"):
        s = 0.5 / np.sqrt(np.where(pos, tr, 1.0))
        q3 = np.stack([0.25 / s, (m[:, 2, 1] - m[:, 1, 2]) * s, (m[:, 0, 2] - m[:, 2, 0]) * s,
                       (m[:, 1, 0] - m[:, 0, 1]) * s], axis=1)
        s0 = 2 * np.sqrt(np.maximum(1 + d[:, 0] - d[:, 1] - d[:, 2], 1e-300))
        q0 = np.stack([(m[:, 2, 1] - m[:, 1, 2]) / s0, 0.25 * s0, (m[:, 0, 1] + m[:, 1, 0]) / s0,
                       (m[:, 0, 2] + m[:, 2, 0]) / s0], axis=1)
        s1 = 2 * np.sqrt(np.maximum(1 + d[:, 1] - d[:, 0] - d[:, 2], 1e-300))
        q1 = np.stack([(m[:, 0, 2] - m[:, 2, 0]) / s1, (m[:, 0, 1] + m[:, 1, 0]) / s1, 0.25 * s1,
                       (m[:, 1, 2] + m[:, 2, 1]) / s1], axis=1)
        s2 = 2 * np.sqrt(np.maximum(1 + d[:, 2] - d[:, 0] - d[:, 1], 1e-300))
        q2 = np.stack([(m[:, 1, 0] - m[:, 0, 1]) / s2, (m[:, 0, 2] + m[:, 2, 0]) / s2,
                       (m[:, 1, 2] + m[:, 2, 1]) / s2, 0.25 * s2], axis=1)
    for b, qb in ((0, q0), (1, q1), (2, q2), (3, q3)):
        q[branch == b] = qb[branch == b]
    return q


def rotate_gaussian(T, gs):
    """gau_io.py:110-126: applies the rotation T to positions and orientations (in place)"""
    T = np.asarray(T, np.float64)
    w, x, y, z = (np.asarray(gs["rot"][:, i], np.float64) for i in range(4))
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]).transpose(2, 0, 1)
    gs["pw"] = (T @ np.asarray(gs["pw"], np.float64).T).T
    gs["rot"] = matrix_to_quaternion(T @ R)
    return gs
