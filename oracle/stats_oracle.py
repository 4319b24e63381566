"""ctypes/numpy front-end of the contribution-statistics oracle (oracle/stats_oracle.c), and its
surfel counterpart in numpy.  TEST INFRASTRUCTURE ONLY.

Per Gaussian, in fp64, over the pixels of one frame: weight_sum = sum of its blending weights
w = tau alpha', weight_max = the largest, hit_count = the pixels with w > 0, and an ambiguity flag
(a threshold decision within `margin` that an fp32 kernel may take the other way, see the C
source).  The colour statistics replay the colour oracle's own binning and front-to-back walk (the
C source includes gs_oracle.c); the surfel statistics reuse surfel_oracle's evaluation, binning and
walk order.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from . import surfel_oracle as so
from .oracle import _f32, _p

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "stats_oracle.c")
_DEPS = (_SRC, os.path.join(_HERE, "gs_oracle.c"))
_lib = None


def _compile(out):
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"  # (as oracle/Makefile)
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.run([gcc, "-O2", "-fopenmp", "-fPIC", "-shared", "-std=c11", "-Wno-unknown-pragmas",
                    "-ffp-contract=off", "-o", out, _SRC, "-lm"], check=True)


def build():
    """Compiles stats_oracle.c next to the colour oracle's library (oracle/_build/), or into a
    temporary directory when the tree is read-only.  -> path of the shared library"""
    so_path = os.path.join(_HERE, "_build", "libgs_oracle_stats.so")
    newest = max(os.path.getmtime(f) for f in _DEPS)
    if os.path.exists(so_path) and os.path.getmtime(so_path) >= newest:
        return so_path
    try:
        _compile(so_path)
        return so_path
    except (OSError, subprocess.CalledProcessError):
        so_path = os.path.join(tempfile.mkdtemp(prefix="gs_oracle_stats_"), "libgs_oracle_stats.so")
        _compile(so_path)
        return so_path


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
    return _lib


def splat_stats(height, width, us, cinv2ds, alphas, fwd, margin=2e-5):
    """orc_draw_stats on the binning of the colour oracle's forward state `fwd` (oracle.splat's or
    rgbd_oracle.splat_rgbd's dict: ranges, gsid).  -> dict(weight_sum[N], weight_max[N] f64,
    hit_count[N] i64, ambiguous[N] bool)"""
    us, cinv2ds = _f32(us), _f32(cinv2ds)
    alphas = _f32(alphas).reshape(-1)
    N = us.shape[0]
    ws, wm = np.zeros(N), np.zeros(N)
    hc = np.zeros(N, np.int64)
    amb = np.zeros(max(N, 1), np.uint8)[:N]
    lib().orc_draw_stats(int(height), int(width), N, _p(fwd["ranges"]), _p(fwd["gsid"]), _p(us), _p(cinv2ds),
                         _p(alphas), _p(ws), _p(wm), _p(hc), _p(amb), C.c_double(margin))
    return dict(weight_sum=ws, weight_max=wm, hit_count=hc, ambiguous=amb.astype(bool))


def surfel_stats(H, W, pre, alphas, bins, margin=2e-5, late_rel=5e-3):
    """The same statistics for surfels: surfel_oracle.render's front-to-back walk (same evaluation,
    skip, stop and clamp) on `pre` (surfel_oracle.preprocess) and bins (surfel_oracle.bin_f32 or
    oracle.bin).  ambiguous: a surfel at a pixel render flags (a threshold, or the G3 / G2 branch,
    within margin) at or after the near decision -- its own, or, for a later surfel, with a weight
    within late_rel of its maximum, as the colour oracle does.
    -> dict(weight_sum[N], weight_max[N], hit_count[N] i64, ambiguous[N] bool)"""
    alphas = np.asarray(alphas, dtype=np.float64).reshape(-1)
    N = len(alphas)
    _, ranges, gsid, _ = bins
    ws, wm = np.zeros(N), np.zeros(N)
    hc = np.zeros(N, np.int64)
    amb_gs = np.zeros(N, bool)
    late = []  # (surfel, its weights at pixels after a near decision)
    for t, X, Y in so._tiles(H, W, ranges):
        Xf, Yf = X.astype(np.float64), Y.astype(np.float64)
        tau = np.ones(len(X))
        amb = np.zeros(len(X), bool)
        for i in gsid[ranges[t, 0]:ranges[t, 1]]:
            e = so._eval(pre["M"][i], pre["u"][i], Xf, Yf)
            ag = alphas[i] * np.exp(-0.5 * e["G"])
            ap = np.minimum(so.ALPHA_CLAMP, ag)
            on = (tau >= so.TAU_STOP) & (ap >= so.ALPHA_SKIP)
            live = tau >= so.TAU_STOP * (1 - margin)
            reach = live & (ap >= so.ALPHA_SKIP * (1 - margin))
            near = live & ((np.abs(ap - so.ALPHA_SKIP) < margin * so.ALPHA_SKIP) | (np.abs(ag - so.ALPHA_CLAMP) < margin) |
                           (np.abs(e["G3"] - e["G2"]) < margin * np.maximum(1.0, e["G2"])))
            near |= (ap >= so.ALPHA_SKIP) & (np.abs(tau - so.TAU_STOP) < margin * so.TAU_STOP)
            near |= amb & (ap >= so.ALPHA_SKIP) & (np.abs(tau - so.TAU_STOP) < late_rel * so.TAU_STOP)
            if (near & reach).any():
                amb_gs[i] = True
            w = np.where(on, tau * ap, 0.0)
            if on.any():
                ws[i] += w.sum()
                wm[i] = max(wm[i], w.max())
                hc[i] += int(on.sum())
                if (amb & on).any():
                    late.append((i, w[amb & on].max()))
            amb |= near
            tau = np.where(on, tau * (1 - ap), tau)
    for i, w in late:
        if w >= (1 - late_rel) * wm[i]:
            amb_gs[i] = True
    return dict(weight_sum=ws, weight_max=wm, hit_count=hc, ambiguous=amb_gs)
