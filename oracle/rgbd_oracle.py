"""ctypes/numpy front-end of the RGB-D oracle (oracle/rgbd_oracle.c).  TEST INFRASTRUCTURE ONLY.

Depth D = sum w z and opacity A = sum w with the image's compositing weights w = tau alpha',
and their backward, in fp64 -- the same arrays and conventions as oracle.splat /
oracle.splat_backward (whose binning it reuses), plus the chain's depth term.  The C source
includes gs_oracle.c, so both libraries take identical threshold decisions.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from .oracle import _f32, _p, bin  # the colour oracle's binning, exactly as its splat() uses it

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "rgbd_oracle.c")
_DEPS = (_SRC, os.path.join(_HERE, "gs_oracle.c"))
_lib = None


def _compile(out):
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"  # (as oracle/Makefile)
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.run([gcc, "-O2", "-fopenmp", "-fPIC", "-shared", "-std=c11", "-Wno-unknown-pragmas",
                    "-ffp-contract=off", "-o", out, _SRC, "-lm"], check=True)


def build():
    """Compiles rgbd_oracle.c next to the colour oracle's library (oracle/_build/), or into a
    temporary directory when the tree is read-only.  -> path of the shared library"""
    so = os.path.join(_HERE, "_build", "libgs_oracle_rgbd.so")
    newest = max(os.path.getmtime(f) for f in _DEPS)
    if os.path.exists(so) and os.path.getmtime(so) >= newest:
        return so
    try:
        _compile(so)
        return so
    except (OSError, subprocess.CalledProcessError):
        so = os.path.join(tempfile.mkdtemp(prefix="gs_oracle_rgbd_"), "libgs_oracle_rgbd.so")
        _compile(so)
        return so


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
    return _lib


def splat_rgbd(height, width, us, cinv2ds, alphas, depths, colors, areas, margin=2e-5):
    """`splat` plus the depth and opacity planes (orc_draw_rgbd): D = sum w z, A = sum w with the
    image's weights w = tau alpha' and z = depths (after the binning's in-place cull, like the
    device op).  depths (f32) and areas (i32) are MODIFIED IN PLACE.  Returns splat's dict plus
    depth[H,W] and alpha[H,W] (f64)."""
    us, cinv2ds, colors = _f32(us), _f32(cinv2ds), _f32(colors)
    alphas = _f32(alphas).reshape(-1)
    H, W = int(height), int(width)
    z = depths.copy()  # the records' depth word is the value before the cull (culled: never drawn)
    P, ranges, gsid, keys = bin(H, W, us, depths, areas)
    L = lib()
    image = np.empty((3, H, W)); contrib = np.empty((H, W), dtype=np.int32)
    ftau = np.empty((H, W)); amb = np.empty((H, W), dtype=np.uint8)
    D = np.empty((H, W)); A = np.empty((H, W))
    L.orc_draw_rgbd(H, W, _p(ranges), _p(gsid), _p(us), _p(cinv2ds), _p(alphas), _p(colors), _p(z),
                    _p(image), _p(D), _p(A), _p(contrib), _p(ftau), _p(amb), C.c_double(margin))
    return dict(image=image, contrib=contrib, final_tau=ftau, ranges=ranges, gsid=gsid, keys=keys,
                ambiguous=amb.astype(bool), P=int(P), depth=D, alpha=A, z=z)


def splat_backward_rgbd(height, width, us, cinv2ds, alphas, colors, depths, fwd, dloss_dgammas,
                        dloss_ddepth, dloss_dalpha, return_ambiguous=False, margin=2e-5):
    """orc_drawB_rgbd on the oracle's own forward state `fwd` (dict from splat_rgbd()); depths: the
    z each Gaussian composited with (fwd["z"]).  -> splat_backward's four arrays + dloss_ddepths[N]
    (+ the bool[N] ambiguity flags)"""
    us, cinv2ds, colors, z = _f32(us), _f32(cinv2ds), _f32(colors), _f32(depths).reshape(-1)
    alphas = _f32(alphas).reshape(-1)
    dl, dld, dla = _f32(dloss_dgammas), _f32(dloss_ddepth), _f32(dloss_dalpha)
    N = us.shape[0]
    du = np.empty((N, 1, 2)); dc = np.empty((N, 1, 3)); da = np.empty((N, 1, 1))
    dcol = np.empty((N, 1, 3)); dz = np.empty(N)
    amb = np.zeros(max(N, 1), dtype=np.uint8)[:N]
    lib().orc_drawB_rgbd(int(height), int(width), N, _p(fwd["ranges"]), _p(fwd["gsid"]), _p(us),
                         _p(cinv2ds), _p(alphas), _p(colors), _p(z), _p(fwd["final_tau"]),
                         _p(fwd["contrib"]), _p(dl), _p(dld), _p(dla), _p(du), _p(dc), _p(da), _p(dcol),
                         _p(dz), _p(amb), C.c_double(margin))
    out = (du, dc, da, dcol, dz)
    return out + (amb.astype(bool),) if return_ambiguous else out


def splat_backward_rgbd_rows(height, width, us, cinv2ds, alphas, colors, depths, fwd, dloss_dgammas, dloss_ddepth,
                             dloss_dalpha, margin=2e-5):
    """The moment rows and dL/dz k_draw_bwd_rgbd writes, in fp64, with their conditioning:
    `oracle.drawB_rows` with the channels (colour, z, 1) against (dL/dimage, dL/dD, dL/dA).
    -> oracle.rows_dict plus ddepths[N], ddepths_abs, ddepths_maha, ddepths_amb"""
    from .oracle import drawB_rows, rows_dict
    H, W = int(height), int(width)
    vals = np.concatenate([_f32(colors).reshape(-1, 3), _f32(depths).reshape(-1, 1),
                           np.ones((len(colors), 1), np.float32)], axis=1)
    dl = np.concatenate([_f32(dloss_dgammas).reshape(3, H, W), _f32(dloss_ddepth).reshape(1, H, W),
                         _f32(dloss_dalpha).reshape(1, H, W)])
    out = rows_dict(drawB_rows(H, W, us, cinv2ds, alphas, vals, fwd, dl, margin))
    for name, a in zip(("ddepths", "ddepths_abs", "ddepths_maha", "ddepths_amb"), out["raw"][:4]):
        out[name] = a[:, 11].copy()
    return out


def chain_depth(Rcw, dloss_ddepths, depths):
    """The depth term of the chain: z = (Rcw pw + tcw)[2], so dL/dpws gains dL/dz Rcw[2,:];
    Gaussians culled for z < 0.2 (depths < 0.2) get 0.  -> [N,3] f64, added to chain_backward's pws."""
    R = np.asarray(Rcw, dtype=np.float64).reshape(3, 3)
    dz = np.asarray(dloss_ddepths, dtype=np.float64).reshape(-1)
    keep = np.asarray(depths, dtype=np.float64).reshape(-1) >= 0.2
    return np.where(keep[:, None], dz[:, None] * R[2][None, :], 0.0)
