"""fp64 model of the bilateral-grid slice, its gradients and the grids' total variation
(easygaussiansplatting_b200/csrc/bilagrid.cu, DESIGN 3.20), plus `torch_slice`, the same slice
composed from torch's F.grid_sample: the independent second formulation the tests compare against.

grids[M, 12, L, Y, X] (channel 4 r + k = A[r][k]); rgb[B, 3, H, W] with B grid indices.  Per pixel:
    g = 0.299 r + 0.587 g + 0.114 b
    (gx, gy, gz) = ((px + 1/2) / W (X - 1), (py + 1/2) / H (Y - 1), clamp(g, 0, 1) (L - 1))
    A = trilinear interpolation of grids[i] there;  out = A[:, :3] rgb + A[:, 3]
"""
import numpy as np

LUMA = np.array([0.299, 0.587, 0.114])


def _axis(coord, n):
    """lower corner, upper corner, fraction of each coordinate on an axis of n points"""
    if n == 1:
        z = np.zeros(np.shape(coord), dtype=np.int64)
        return z, z, np.zeros(np.shape(coord))
    i0 = np.minimum(np.floor(coord).astype(np.int64), n - 2)
    return i0, i0 + 1, coord - i0


def _as_batch(rgb, ids):
    rgb = np.asarray(rgb, dtype=np.float64)
    if rgb.ndim == 3:
        rgb = rgb[None]
    ids = [int(ids)] if np.ndim(ids) == 0 else [int(i) for i in ids]
    assert len(ids) == rgb.shape[0]
    return rgb, ids


def slice_grids(grids, rgb, ids, dout=None, amb_eps=1e-5):
    """-> dict with out [B,3,H,W]; with dout [B,3,H,W] also drgb, dgrids [M,12,L,Y,X],
    dgrids_cond (per entry: the sum of |terms| added into it) and dgrids_cond_t (per entry: the sum
    over its terms of |d term / d t| for t = tx, ty, tz, with tz's scaled by (L - 1) (1 + sum_k
    luma_k |rgb_k|) and tx's, ty's by X - 1, Y - 1: how far the entry moves when the pixel's
    coordinates carry a relative rounding error, which dominates for large grids); ambiguous [B,H,W]: pixels whose
    unclamped g (L - 1) lies within amb_eps of an integer (a level or a clamp bound), where dL/drgb
    jumps between fp32 and fp64 while out and dL/dgrids stay continuous."""
    G = np.asarray(grids, dtype=np.float64)
    M, _, L, Y, X = G.shape
    rgb, ids = _as_batch(rgb, ids)
    B, _, H, W = rgb.shape
    x0, x1, tx = _axis((np.arange(W) + 0.5) / W * (X - 1), X)
    y0, y1, ty = _axis((np.arange(H) + 0.5) / H * (Y - 1), Y)
    res = {"out": np.zeros_like(rgb), "ambiguous": np.zeros((B, H, W), dtype=bool)}
    if dout is not None:
        dout = np.asarray(dout, dtype=np.float64).reshape(rgb.shape)
        res.update(drgb=np.zeros_like(rgb), dgrids=np.zeros_like(G), dgrids_cond=np.zeros_like(G),
                   dgrids_cond_t=np.zeros_like(G))
    xs = ((x0, 1.0 - tx), (x1, tx))
    ys = ((y0, 1.0 - ty), (y1, ty))
    for b in range(B):
        Gi = G[ids[b]]
        v = np.concatenate([rgb[b], np.ones((1, H, W))])  # [rgb, 1]
        g = np.tensordot(LUMA, rgb[b], axes=1)
        gu = g * (L - 1)
        if L > 1:
            res["ambiguous"][b] = np.abs(gu - np.round(gu)) < amb_eps
        z0, z1, tz = _axis(np.clip(g, 0.0, 1.0) * (L - 1), L)
        A = np.zeros((12, H, W))
        dA = np.zeros((12, H, W))  # dA/dgz
        corners = []
        for xi, wx in xs:
            for yi, wy in ys:
                wxy = wy[:, None] * wx[None, :]
                yy, xx = np.broadcast_to(yi[:, None], (H, W)), np.broadcast_to(xi[None, :], (H, W))
                c0, c1 = Gi[:, z0, yy, xx], Gi[:, z1, yy, xx]
                A += wxy * ((1.0 - tz) * c0 + tz * c1)
                dA += wxy * (c1 - c0)
                # |d w / d (tx, ty, tz)| of the corner, each scaled by its coordinate's rounding
                sxy = np.abs(wy)[:, None] * (X - 1) + np.abs(wx)[None, :] * (Y - 1)
                sz = wxy * (L - 1) * (1.0 + np.tensordot(LUMA, np.abs(rgb[b]), axes=1))
                corners += [(xx, yy, z0, wxy * (1.0 - tz), sxy + sz), (xx, yy, z1, wxy * tz, sxy + sz)]
        A3 = A.reshape(3, 4, H, W)
        res["out"][b] = np.einsum("rkhw,khw->rhw", A3, v)
        if dout is None:
            continue
        d = dout[b]
        drgb = np.einsum("rkhw,rhw->khw", A3[:, :3], d)
        if L > 1:
            s = np.einsum("rhw,rkhw,khw->hw", d, dA.reshape(3, 4, H, W), v) * (L - 1)
            s = np.where((g > 0.0) & (g < 1.0), s, 0.0)
            drgb += LUMA[:, None, None] * s
        res["drgb"][b] = drgb
        size = 12 * L * Y * X
        for xx, yy, zz, w, sens in corners:
            for r in range(3):
                for k in range(4):
                    c = 4 * r + k
                    dv = d[r] * v[k]
                    t = (w * dv).ravel()
                    flat = (((c * L + zz) * Y + yy) * X + xx).ravel()
                    res["dgrids"][ids[b]] += np.bincount(flat, t, size).reshape(12, L, Y, X)
                    res["dgrids_cond"][ids[b]] += np.bincount(flat, np.abs(t), size).reshape(12, L, Y, X)
                    res["dgrids_cond_t"][ids[b]] += np.bincount(flat, (sens * np.abs(dv)).ravel(),
                                                                size).reshape(12, L, Y, X)
    return res


def total_variation(grids):
    """-> (TV, dTV/dgrids): TV = sum over the axes L, Y, X of mean((shifted - grids)^2), the mean over
    every difference along the axis; an axis of size 1 adds 0"""
    G = np.asarray(grids, dtype=np.float64)
    tv, grad = 0.0, np.zeros_like(G)
    for ax in (2, 3, 4):
        n = G.shape[ax]
        if n == 1:
            continue
        d = np.diff(G, axis=ax)
        tv += (d * d).sum() / d.size
        g2 = 2.0 * d / d.size
        pad = [(0, 0)] * 5
        pad[ax] = (1, 0)
        grad += np.pad(g2, pad)  # d/d(later element) of its difference
        pad[ax] = (0, 1)
        grad -= np.pad(g2, pad)  # d/d(earlier element)
    return tv, grad


def torch_slice(grids, rgb, ids):
    """The slice composed from F.grid_sample (any dtype and device): rgb [3,H,W] or [B,3,H,W] ->
    out shaped like rgb; differentiable by autograd in grids and rgb."""
    import torch
    import torch.nn.functional as F
    single = rgb.dim() == 3
    rgb4 = rgb[None] if single else rgb
    ids = [int(ids)] if np.ndim(ids) == 0 else [int(i) for i in ids]
    B, _, H, W = rgb4.shape
    dev, dt = rgb4.device, rgb4.dtype
    xs = ((torch.arange(W, device=dev, dtype=dt) + 0.5) / W).view(1, W).expand(H, W)
    ys = ((torch.arange(H, device=dev, dtype=dt) + 0.5) / H).view(H, 1).expand(H, W)
    outs = []
    for b in range(B):
        g = 0.299 * rgb4[b, 0] + 0.587 * rgb4[b, 1] + 0.114 * rgb4[b, 2]
        xyz = torch.stack([xs, ys, g], dim=-1) * 2.0 - 1.0
        A = F.grid_sample(grids[ids[b]:ids[b] + 1], xyz.view(1, 1, H, W, 3), mode="bilinear",
                          padding_mode="border", align_corners=True).view(3, 4, H, W)
        outs.append((A[:, :3] * rgb4[b][None]).sum(1) + A[:, 3])
    out = torch.stack(outs)
    return out[0] if single else out
