"""ctypes/numpy front-end of the absolute-gradient oracle (oracle/absgrad_oracle.c).  TEST
INFRASTRUCTURE ONLY.

The per-pixel absolute sums of dL/du that AbsGS densifies on, in fp64, on the colour oracle's or
the RGB-D oracle's own forward state (oracle.splat / rgbd_oracle.splat_rgbd): the same arrays and
conventions as oracle.splat_backward / rgbd_oracle.splat_backward_rgbd.  The C source includes
gs_oracle.c and rgbd_oracle.c, so all three libraries take identical threshold decisions.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from .oracle import _f32, _p

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "absgrad_oracle.c")
_DEPS = (_SRC, os.path.join(_HERE, "rgbd_oracle.c"), os.path.join(_HERE, "gs_oracle.c"))
_lib = None


def _compile(out):
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"  # (as oracle/Makefile)
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.run([gcc, "-O2", "-fopenmp", "-fPIC", "-shared", "-std=c11", "-Wno-unknown-pragmas",
                    "-ffp-contract=off", "-o", out, _SRC, "-lm"], check=True)


def build():
    """Compiles absgrad_oracle.c next to the colour oracle's library (oracle/_build/), or into a
    temporary directory when the tree is read-only.  -> path of the shared library"""
    so = os.path.join(_HERE, "_build", "libgs_oracle_absgrad.so")
    newest = max(os.path.getmtime(f) for f in _DEPS)
    if os.path.exists(so) and os.path.getmtime(so) >= newest:
        return so
    try:
        _compile(so)
        return so
    except (OSError, subprocess.CalledProcessError):
        so = os.path.join(tempfile.mkdtemp(prefix="gs_oracle_absgrad_"), "libgs_oracle_absgrad.so")
        _compile(so)
        return so


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
    return _lib


def splat_backward_abs(height, width, us, cinv2ds, alphas, colors, fwd, dloss_dgammas, margin=2e-5):
    """orc_drawB_abs on the colour oracle's forward state `fwd` (dict from oracle.splat()).
    -> (dloss_dus[N,2] signed sums, dloss_dus_abs[N,2] absolute sums, bool[N] ambiguity flags), f64"""
    us, cinv2ds, colors = _f32(us), _f32(cinv2ds), _f32(colors)
    alphas, dl = _f32(alphas).reshape(-1), _f32(dloss_dgammas)
    N = us.shape[0]
    du = np.empty((N, 2)); dabs = np.empty((N, 2))
    amb = np.zeros(max(N, 1), dtype=np.uint8)[:N]
    lib().orc_drawB_abs(int(height), int(width), N, _p(fwd["ranges"]), _p(fwd["gsid"]), _p(us), _p(cinv2ds),
                        _p(alphas), _p(colors), _p(fwd["final_tau"]), _p(fwd["contrib"]), _p(dl), _p(du), _p(dabs),
                        _p(amb), C.c_double(margin))
    return du, dabs, amb.astype(bool)


def splat_backward_abs_rows(height, width, us, cinv2ds, alphas, colors, fwd, dloss_dgammas, depths=None,
                            dloss_ddepth=None, dloss_dalpha=None, margin=2e-5):
    """The absolute sums of k_draw_bwd_abs (given depths and the two planes, k_draw_bwd_rgbd_abs) next to
    their moment rows, in fp64, with their conditioning.  -> the dict of `oracle.splat_backward_rows`
    (`rgbd_oracle.splat_backward_rgbd_rows`) plus dus_abs[N,2], dus_abs_abs, dus_abs_maha, dus_abs_amb.
    Every term of dus_abs is >= 0; dus_abs_abs also counts the cancellation inside A dx + B dy."""
    from . import oracle as orc
    from . import rgbd_oracle as org
    if depths is None:
        out = orc.splat_backward_rows(height, width, us, cinv2ds, alphas, colors, fwd, dloss_dgammas, margin)
    else:
        out = org.splat_backward_rgbd_rows(height, width, us, cinv2ds, alphas, colors, depths, fwd, dloss_dgammas,
                                           dloss_ddepth, dloss_dalpha, margin)
    for name, a in zip(("dus_abs", "dus_abs_abs", "dus_abs_maha", "dus_abs_amb"), out["raw"][:4]):
        out[name] = a[:, 6:8].copy()
    return out


def splat_backward_rgbd_abs(height, width, us, cinv2ds, alphas, colors, depths, fwd, dloss_dgammas, dloss_ddepth,
                            dloss_dalpha, margin=2e-5):
    """orc_drawB_rgbd_abs on the RGB-D oracle's forward state `fwd` (dict from
    rgbd_oracle.splat_rgbd()); depths: the z each Gaussian composited with (fwd["z"]).
    -> (dloss_dus[N,2], dloss_dus_abs[N,2], bool[N] ambiguity flags), f64"""
    us, cinv2ds, colors, z = _f32(us), _f32(cinv2ds), _f32(colors), _f32(depths).reshape(-1)
    alphas = _f32(alphas).reshape(-1)
    dl, dld, dla = _f32(dloss_dgammas), _f32(dloss_ddepth), _f32(dloss_dalpha)
    N = us.shape[0]
    du = np.empty((N, 2)); dabs = np.empty((N, 2))
    amb = np.zeros(max(N, 1), dtype=np.uint8)[:N]
    lib().orc_drawB_rgbd_abs(int(height), int(width), N, _p(fwd["ranges"]), _p(fwd["gsid"]), _p(us), _p(cinv2ds),
                             _p(alphas), _p(colors), _p(z), _p(fwd["final_tau"]), _p(fwd["contrib"]), _p(dl),
                             _p(dld), _p(dla), _p(du), _p(dabs), _p(amb), C.c_double(margin))
    return du, dabs, amb.astype(bool)
