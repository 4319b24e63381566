"""Mesh extraction from depth maps (DESIGN 3.17): a dense TSDF volume on the GPU, fused from the
depth maps a trained model renders and turned into a triangle mesh by marching cubes.

    vol = TSDFVolume(lo, hi, voxel_size)          # trunc = 5 voxels, no depth cut, with colour
    vol.integrate(depth[V, H, W], cams, color[V, 3, H, W])
    verts, faces, colors = vol.extract()
    gau_io.save_mesh_ply("mesh.ply", verts, faces, colors)

INTEGRATION.md gives the 2D Gaussian Splatting recipe (median depth, alpha mask, batches).
"""
import math

import torch

from . import ops


class TSDFVolume:
    """A grid of sample points from lo, voxel_size apart, covering [lo, hi] on every axis
    (n = ceil((hi - lo) / voxel_size) + 1 points per axis): tsdf [nz, ny, nx] (1 when new),
    weight (0) and, with color=True, color [3, nz, ny, nx] (0).  trunc: the truncation distance
    (default 5 voxels, as 2D Gaussian Splatting uses); depth_trunc: depths beyond it are not fused.
    The colour grid makes the volume 2.5x as large."""

    def __init__(self, lo, hi, voxel_size, trunc=None, depth_trunc=math.inf, color=True, device=None):
        lo, hi = [float(x) for x in lo], [float(x) for x in hi]
        if len(lo) != 3 or len(hi) != 3:
            raise ValueError("lo and hi must have 3 values")
        if not all(math.isfinite(x) for x in lo + hi) or not all(h > l for l, h in zip(lo, hi)):
            raise ValueError("lo and hi must be finite with hi > lo on every axis")
        self.voxel_size = float(voxel_size)
        if not (math.isfinite(self.voxel_size) and self.voxel_size > 0):
            raise ValueError("voxel_size must be finite and > 0")
        self.trunc = 5 * self.voxel_size if trunc is None else float(trunc)
        if not (math.isfinite(self.trunc) and self.trunc > 0):
            raise ValueError("trunc must be finite and > 0")
        self.depth_trunc = float(depth_trunc)
        if not self.depth_trunc > 0:
            raise ValueError("depth_trunc must be > 0")
        # a span that is a whole number of voxels up to rounding gets no extra plane
        dims = [math.ceil((h - l) / self.voxel_size - 1e-6) + 1 for l, h in zip(lo, hi)]
        if math.prod(dims) >= 2 ** 31:
            raise ValueError("the grid has %d x %d x %d = 2^31 or more points" % tuple(dims))
        self.origin = lo
        self.dims = tuple(dims)  # (nx, ny, nz)
        nx, ny, nz = dims
        dev = torch.device("cuda") if device is None else torch.device(device)
        self.tsdf = torch.ones((nz, ny, nx), dtype=torch.float32, device=dev)
        self.weight = torch.zeros((nz, ny, nx), dtype=torch.float32, device=dev)
        self.color = torch.zeros((3, nz, ny, nx), dtype=torch.float32, device=dev) if color else None

    def integrate(self, depth, cams, color=None):
        """Fuses depth [H, W] seen by one camera, or [V, H, W] by a list of V cameras, in order.
        Pinhole cameras only, each with the depth map's width and height.  color: [3, H, W] /
        [V, 3, H, W] in [0, 1], used when the volume has colour (then required)."""
        single = depth.dim() == 2
        if single:
            depth, cams = depth[None], [cams]
            color = None if color is None else color[None]
        cams = list(cams) if isinstance(cams, (list, tuple)) else [cams]
        if depth.dim() != 3 or len(cams) != depth.shape[0]:
            raise ValueError("depth must be [H, W] with one camera or [V, H, W] with V cameras")
        H, W = depth.shape[1:]
        for k, c in enumerate(cams):
            if getattr(c, "camera_model", "pinhole") != "pinhole":
                raise ValueError("camera %d: TSDF fusion takes pinhole cameras only, got camera_model=%r"
                                 % (k, c.camera_model))
            if (int(c.width), int(c.height)) != (W, H):
                raise ValueError("camera %d is %dx%d but the depth map is %dx%d" % (k, c.width, c.height, W, H))
        if (color is None) != (self.color is None):
            raise ValueError("this volume %s colour" % ("needs" if self.color is not None else "has no"))
        table = ops.camera_table(cams, device=self.tsdf.device)
        ops.tsdf_integrate(self.tsdf, self.weight, self.color, self.origin, self.voxel_size, self.trunc,
                           self.depth_trunc, table, depth, color)

    def extract(self):
        """-> (verts[V, 3] float32, faces[F, 3] int32, colors[V, 3] float32 or None), on the device"""
        return ops.tsdf_extract(self.tsdf, self.weight, self.color, self.origin, self.voxel_size)
