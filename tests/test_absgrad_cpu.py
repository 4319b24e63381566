"""CPU checks of absolute-gradient densification (AbsGS): the fp64 oracle's per-pixel absolute sums
of dL/du against the colour and RGB-D oracles' signed sums, on synthetic scenes and on hand-built
frames where the two must agree exactly; the two new entry points' ctypes signatures and argument
errors; and the two _abs rasterizers in the sm_90a binary."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import absgrad_oracle as oabs
from oracle import oracle as orc
from oracle import rgbd_oracle as orgbd
from easygaussiansplatting_b200.scene import upstream_gradient

from test_rgbd_cpu import _scene64, _stages

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _frame(N, W, H, seed):
    sc = _scene64(N, W, H, seed=seed)
    us, ci, col, d32, areas, _ = _stages(sc, W, H)
    return us, ci, col, d32, areas, sc["alphas"]


@pytest.mark.parametrize("N,W,H,seed", [(600, 97, 61, 3), (1500, 128, 80, 11)])
def test_signed_sums_equal_the_colour_oracle_and_bound_the_absolute_sums(N, W, H, seed):
    us, ci, col, d32, areas, al = _frame(N, W, H, seed)
    f = orc.splat(H, W, us, ci, al, d32, col, areas)
    dl = upstream_gradient(W, H, seed).astype(np.float64) * (3.0 * W * H)
    du_ref, _, _, _, amb_ref = orc.splat_backward(H, W, us, ci, al, col, f, dl, return_ambiguous=True)
    du, dabs, amb = oabs.splat_backward_abs(H, W, us, ci, al, col, f, dl)
    du_ref = du_ref.reshape(N, 2)
    # (the oracles sum with OpenMP atomics: order-level differences)
    assert np.abs(du - du_ref).max() <= 1e-12 * np.abs(du_ref).max()
    assert np.array_equal(amb, amb_ref)
    assert np.all(dabs >= np.abs(du) - 1e-12 * np.abs(du).max())
    # cancellation is real on a textured upstream gradient: the statistic is much larger in total
    assert dabs.sum() > 2.0 * np.abs(du).sum()
    # exact zeros where no pixel replays the Gaussian (culled, off-screen, or never above 0.002)
    touched = np.zeros(N, bool)
    touched[np.unique(f["gsid"])] = True
    assert (~touched).any() and not dabs[~touched].any() and not du[~touched].any()


def test_rgbd_signed_sums_equal_the_rgbd_oracle():
    N, W, H = 700, 83, 57
    us, ci, col, d32, areas, al = _frame(N, W, H, 5)
    g = orgbd.splat_rgbd(H, W, us, ci, al, d32, col, areas)
    dl = upstream_gradient(W, H, 5).astype(np.float64) * (3.0 * W * H)
    rng = np.random.default_rng(9)
    dld = rng.normal(size=(H, W)).astype(np.float32)
    dla = rng.normal(size=(H, W)).astype(np.float32)
    zero = np.zeros((H, W), np.float32)
    for a, b, c in ((dl, dld, dla), (dl * 0, dld, zero), (dl * 0, zero, dla)):
        ref = orgbd.splat_backward_rgbd(H, W, us, ci, al, col, g["z"], g, a, b, c)
        du, dabs, _ = oabs.splat_backward_rgbd_abs(H, W, us, ci, al, col, g["z"], g, a, b, c)
        du_ref = ref[0].reshape(N, 2)
        assert np.abs(du - du_ref).max() <= 1e-12 * np.abs(du_ref).max()
        assert np.all(dabs >= np.abs(du) - 1e-12 * np.abs(du).max())
        assert dabs.max() > 0  # depth-only and alpha-only upstream gradients reach the statistic
    # with dL/dD = dL/dA = 0 the RGB-D form is the colour form
    f = dict(g)
    du3, dabs3, _ = oabs.splat_backward_abs(H, W, us, ci, al, col, f, dl)
    du5, dabs5, _ = oabs.splat_backward_rgbd_abs(H, W, us, ci, al, col, g["z"], g, dl, zero, zero)
    assert np.abs(du3 - du5).max() <= 1e-12 * np.abs(du3).max()
    assert np.abs(dabs3 - dabs5).max() <= 1e-12 * np.abs(dabs3).max()


def _hand_frame():
    """32x24 frame, axis-aligned conics (B = 0), positive colours and upstream gradient:
    g0 reaches one pixel only (tiny footprint at (5.3, 7.2)); g1 is centred above-left of every
    pixel, so each of its per-pixel terms has dx < 0, dy < 0 and w > 0 (it is the farthest: its
    dL/dalpha' is tau c . dl > 0); g2 is off-screen; g3 never reaches alpha' = 0.002."""
    W, H = 32, 24
    us = np.array([[5.3, 7.2], [-0.5, -0.5], [-100.0, -100.0], [20.0, 12.0]], np.float32)
    ci = np.array([[20.0, 0.0, 20.0], [0.05, 0.0, 0.08], [1.0, 0.0, 1.0], [0.1, 0.0, 0.1]], np.float32)
    al = np.array([0.2, 0.7, 0.5, 0.0015], np.float32)
    col = np.array([[0.3, 0.2, 0.1], [0.9, 0.8, 0.7], [0.5, 0.5, 0.5], [0.5, 0.5, 0.5]], np.float32)
    depths = np.array([2.0, 3.0, 4.0, 5.0], np.float32)
    areas = np.array([[3, 3], [12, 12], [4, 4], [10, 10]], np.int32)
    dl = np.full((3, H, W), 1e-3, np.float32)
    return W, H, us, ci, al, col, depths, areas, dl


def test_equality_for_one_pixel_and_same_sign_terms_and_zeros():
    W, H, us, ci, al, col, depths, areas, dl = _hand_frame()
    f = orc.splat(H, W, us, ci, al, depths, col, areas)
    du, dabs, _ = oabs.splat_backward_abs(H, W, us, ci, al, col, f, dl)
    # g0: one replayed pixel, g1: terms of one sign per component -> |sum| == sum |.|
    for g in (0, 1):
        assert np.all(np.abs(du[g]) > 0)
        assert np.allclose(dabs[g], np.abs(du[g]), rtol=1e-15, atol=0), (g, dabs[g], du[g])
    assert not dabs[2].any() and not dabs[3].any() and not du[2].any() and not du[3].any()
    # g0 really is one pixel: the other pixels around it stay below the skip threshold
    A = float(ci[0, 0])
    ap = [al[0] * np.exp(-0.5 * A * ((us[0, 0] - x) ** 2 + (us[0, 1] - y) ** 2))
          for x in range(W) for y in range(H)]
    assert sum(a >= 0.002 for a in ap) == 1
    # the RGB-D form on the same frame with only a depth gradient: same identities
    g = orgbd.splat_rgbd(H, W, us, ci, al, np.array([2.0, 3.0, 4.0, 5.0], np.float32), col, areas.copy())
    zero = np.zeros((H, W), np.float32)
    du5, dabs5, _ = oabs.splat_backward_rgbd_abs(H, W, us, ci, al, col, g["z"], g, dl * 0, zero + 1e-3, zero)
    assert np.allclose(dabs5[1], np.abs(du5[1]), rtol=1e-15, atol=0) and np.all(dabs5[1] > 0)
    assert np.allclose(dabs5[0], np.abs(du5[0]), rtol=1e-15, atol=0)
    assert not dabs5[2:].any()


# ---------------------------------------------------------------- ABI and binary
def _header_args(name):
    src = open(os.path.join(ROOT, "include", "gsplat_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    m = re.search(r"\b%s\s*\(([^)]*)\)" % name, src)
    return [a.strip() for a in m.group(1).split(",")]


def test_abs_entry_points_signatures_and_argument_errors():
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    lib = _lib.load()
    for base in ("gsb_splat_backward", "gsb_splat_backward_rgbd"):
        plain, new = _header_args(base), _header_args(base + "_abs")
        # the plain call's arguments, then float *dloss_dus_abs, then the stream
        assert new[:-2] == plain[:-1] and new[-1] == plain[-1] and new[-2] == "float *dloss_dus_abs"
        res, args = _lib.SIGNATURES[base + "_abs"]
        pres, pargs = _lib.SIGNATURES[base]
        assert res is pres and args == pargs[:-1] + [C.c_void_p, C.c_void_p] and len(args) == len(new)
    vp = C.c_void_p
    plain = [vp(256)] * 9
    # N > 0 without the output is an argument error; N == 0 writes nothing and needs no device
    rc = lib.gsb_splat_backward_abs(16, 16, 10, 0, *plain, None, vp(256), 1 << 20, None, None, None, None, vp(256),
                                    None, None)
    assert rc != 0 and b"null dloss_dus_abs" in lib.gsb_last_error()
    rc = lib.gsb_splat_backward_rgbd_abs(16, 16, 10, 0, *([vp(256)] * 12), None, vp(256), 1 << 20, None, None, None,
                                         None, vp(256), vp(256), None, None)
    assert rc != 0 and b"null dloss_dus_abs" in lib.gsb_last_error()
    assert lib.gsb_splat_backward_abs(16, 16, 0, 0, *([None] * 11), 0, *([None] * 7)) == 0
    assert lib.gsb_splat_backward_rgbd_abs(16, 16, 0, 0, *([None] * 14), 0, *([None] * 8)) == 0
    assert lib.gsb_abi_version() == 1
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    assert names[-5:] == ["draw_backward_abs", "draw_backward_rgbd_abs", "adam", "draw_rgbd", "draw_backward_rgbd"]


def test_abs_rasterizers_are_sm90a_with_cp_async_record_gather():
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    for name in ("k_draw_bwd_abs", "k_draw_bwd_rgbd_abs"):
        body = [f for f in funcs if f.startswith("_ZN3gsb%d%sE" % (len(name), name))]
        assert len(body) == 1, name
        for op in ("LDGSTS.E.BYPASS.128", "LDGDEPBAR", "DEPBAR.LE", "MUFU.EX2", "REDG.E.ADD.F32"):
            assert op in body[0], "%s: %s missing" % (name, op)
    r = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True)
    found = re.findall(r"Function (_ZN3gsb\d+k_draw_bwd\w*_abs\w*):\s*\n\s*(REG:.*)", r.stdout)
    assert len(found) == 2, found
    for name, usage in found:  # built for 5 CTAs/SM (DESIGN 3.13): 96 registers, a small stack
        assert "REG:96 " in usage and "LOCAL:0 " in usage, (name, usage)
        assert int(re.search(r"STACK:(\d+)", usage).group(1)) <= 32, (name, usage)
