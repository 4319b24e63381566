"""Batched rendering without a GPU (DESIGN 3.21): the batch entry points' argument errors come back
before any launch, the workspace queries take C, the cameras of a batch must agree on what they
share, the profile ids of the batch kernels, and a host build of the tall frame's rectangle arithmetic
(rect_math.h) against a numpy model of the single frame's rectangle, offset per camera."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from easygaussiansplatting_b200 import _lib, build, ops
from easygaussiansplatting_b200.gsfunction import Camera

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def _err(lib):
    return lib.gsb_last_error().decode()


def test_batch_workspace_queries_take_C(lib):
    one = lib.gsb_splat_batch_workspace_bytes(1, 1000, 61, 83, 5000)
    assert one == lib.gsb_splat_workspace_bytes(1000, 64, 83, 5000)  # one frame padded to whole tiles
    assert lib.gsb_splat_batch_workspace_bytes(8, 1000, 61, 83, 5000) > one
    assert lib.gsb_splat_bin_batch_workspace_bytes(8, 1000) == lib.gsb_splat_bin_workspace_bytes(8000)
    assert lib.gsb_splat_backward_batch_workspace_bytes(8, 1000, 61, 83, 0) > \
        lib.gsb_splat_backward_batch_workspace_bytes(1, 1000, 61, 83, 0)
    assert lib.gsb_splat_batch_records_offset(3, 100, 61, 83, 10) % 256 == 0
    # what the entry points refuse sizes nothing (no int overflow of C N)
    for Cn, N in ((0, 1000), (-1, 1000), (2, 1 << 30), (64, 1 << 26), (1, -1)):
        assert lib.gsb_splat_bin_batch_workspace_bytes(Cn, N) == 0
        assert lib.gsb_splat_batch_workspace_bytes(Cn, N, 61, 83, 10) == 0
        assert lib.gsb_splat_batch_records_offset(Cn, N, 61, 83, 10) == 0
        assert lib.gsb_splat_backward_batch_workspace_bytes(Cn, N, 61, 83, 0) == 0


def test_batch_argument_errors_before_any_launch(lib):
    P, dk = C.c_int64(0), C.c_uint32(0)
    ws = (C.c_char * 4096)()
    bin_ws = C.addressof(ws) + (-C.addressof(ws)) % 16
    # C < 1, C N >= 2^31, C gy > GSB_MAX_GRID_TILES
    assert lib.gsb_splat_bin_batch(0, 16, 16, 10, None, None, None, bin_ws, 4096, C.byref(P), C.byref(dk), None) != 0
    assert "C < 1" in _err(lib)
    assert lib.gsb_splat_bin_batch(2, 16, 16, 1 << 30, None, None, None, bin_ws, 1 << 40, C.byref(P), C.byref(dk),
                                   None) != 0
    assert "2^31" in _err(lib)
    assert lib.gsb_splat_bin_batch(64, 16 * 1100, 16, 10, None, None, None, bin_ws, 1 << 40, C.byref(P), C.byref(dk),
                                   None) != 0
    assert "65535" in _err(lib)
    assert lib.gsb_splat_bin_batch(2, 16, 16, 10, None, None, None, bin_ws + 4, 1 << 40, C.byref(P), C.byref(dk),
                                   None) != 0
    assert "misaligned" in _err(lib)
    # 2^30 patches or more
    args = [None] * 8 + [0] + [None] * 6
    assert lib.gsb_splat_render_batch(2, 16, 16, 10, 1 << 30, 0, *args) != 0
    assert "2^30" in _err(lib)
    fwd = [None] * 7 + [1 << 30, 0, bin_ws, 1 << 40, None, 0] + [None] * 7
    assert lib.gsb_splat_forward_batch(2, 16, 16, 10, *fwd) != 0
    assert "P_cap" in _err(lib)
    assert lib.gsb_splat_backward_batch(0, 16, 16, 10, 0, *([None] * 11), 0, None, None) != 0
    assert "C < 1" in _err(lib)
    # the per-Gaussian entry points: C, camera count, model checks per camera
    intr_rows = (C.c_float * 16)(200.0, 200.0, 8.0, 8.0, 0, 0, 0, 0, -1.0, 200.0, 8.0, 8.0, 0, 0, 0, 0)
    intr = C.addressof(intr_rows)  # host memory
    base = [None] * 5  # pws, rots, scales, shs, poses
    outs = [None] * 8 + [None]
    assert lib.gsb_preprocess_forward_batch(0, 10, 16, *base, intr, 0, 16.0, 16.0, *outs) != 0
    assert "C < 1" in _err(lib)
    assert lib.gsb_preprocess_forward_batch(65, 10, 16, *base, intr, 0, 16.0, 16.0, *outs) != 0
    assert "GSB_BATCH_MAX_CAMERAS" in _err(lib)
    assert lib.gsb_preprocess_forward_batch(2, 1 << 30, 16, *base, intr, 0, 16.0, 16.0, *outs) != 0
    assert "2^31" in _err(lib)
    assert lib.gsb_preprocess_forward_batch(2, 10, 16, *base, intr, 2, 16.0, 16.0, *outs) != 0  # fisheye, fx < 0
    assert "fx and fy must be > 0" in _err(lib)
    assert lib.gsb_preprocess_forward_batch(2, 10, 16, *base, intr, 3, 16.0, 16.0, *outs) != 0
    assert "unknown camera model" in _err(lib)
    assert lib.gsb_preprocess_backward_batch(2, 10, 16, *base, intr, 4, 16.0, 16.0, *([None] * 11)) != 0
    assert "fx and fy must be > 0" in _err(lib)
    ok_rows = (C.c_float * 8)(200.0, 200.0, 8.0, 8.0, 0, 0, 0, 0)
    ok = C.addressof(ok_rows)
    rec = bin_ws + 8
    assert lib.gsb_preprocess_forward_batch(1, 10, 16, *base, ok, 0, 16.0, 16.0, *([None] * 6), rec, None, None) != 0
    assert "records misaligned" in _err(lib)


def test_batch_profile_ids(lib):
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    for n in ("rects+scan_batch", "preprocess_forward_batch", "preprocess_backward_batch", "draw_batch",
              "draw_rgbd_batch", "draw_backward_batch", "draw_backward_rgbd_batch"):
        assert n in names


def test_batch_cameras_must_share_size_model_and_antialiasing():
    R, t = torch.eye(3), torch.zeros(3)
    cams = [Camera(64, 48, 50.0, 50.0, 32.0, 24.0, R, t), Camera(64, 48, 55.0, 52.0, 31.0, 25.0, R, t)]
    bc = ops.BatchCameras(cams, "cpu")
    assert bc.C == 2 and bc.poses.shape == (2, 15) and bc.intrinsics.shape == (2, ops.BATCH_INTRINSICS_ROW)
    assert bc.intrinsics[1, :4].tolist() == [55.0, 52.0, 31.0, 25.0]
    for other in (Camera(64, 40, 50.0, 50.0, 32.0, 24.0, R, t), Camera(60, 48, 50.0, 50.0, 32.0, 24.0, R, t),
                  Camera(64, 48, 50.0, 50.0, 32.0, 24.0, R, t, antialiased=True),
                  Camera(64, 48, 50.0, 50.0, 32.0, 24.0, R, t, camera_model="fisheye")):
        with pytest.raises(ValueError, match="share"):
            ops.BatchCameras([cams[0], other], "cpu")
    with pytest.raises(ValueError, match="1 to 64"):
        ops.BatchCameras([], "cpu")
    with pytest.raises(ValueError, match="1 to 64"):
        ops.BatchCameras(cams * 33, "cpu")


# ---------------------------------------------------------------- the tall frame's rectangles
RECT_SO = os.path.join(HERE, "host_shim", "_build", "librect_host.so")


@pytest.fixture(scope="module")
def rect_shim():
    src = os.path.join(HERE, "host_shim", "rect_host.cpp")
    hdr = os.path.join(HERE, "..", "easygaussiansplatting_b200", "csrc", "rect_math.h")
    os.makedirs(os.path.dirname(RECT_SO), exist_ok=True)
    if not os.path.exists(RECT_SO) or os.path.getmtime(RECT_SO) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", RECT_SO, src],
                       check=True)
    return C.CDLL(RECT_SO)


def _single_rect_model(u, r, gx, gy):
    """numpy float32 model of one frame's rectangle (reference kernel.cu:105-110): [N,4] x0, x1, y0, y1"""
    f = np.float32
    u, r = u.astype(f), r.astype(f)
    lo = np.trunc((u - r) / f(16)).astype(np.int64)
    hi = np.trunc((((u + r) + f(16)) - f(1)) / f(16)).astype(np.int64)
    g = np.array([gx, gy])
    lo, hi = np.clip(lo, 0, g), np.clip(hi, 0, g)
    return np.stack([lo[:, 0], hi[:, 0], lo[:, 1], hi[:, 1]], 1)


@pytest.mark.parametrize("W,H", [(83, 61), (1920, 1080), (100, 17)])
@pytest.mark.parametrize("Cn", [1, 2, 7])
def test_tall_frame_rectangles_are_the_single_frames_offset(rect_shim, Cn, W, H):
    """record c N + n: the single frame's rectangle of camera c, clamped to its own gy rows and moved down
    by c gy -- at frame edges (means within a radius of every border, outside, exactly on tile lines),
    with zero, small and huge radii, at H % 16 != 0"""
    rng = np.random.default_rng(Cn * 1000 + W)
    N = 4000
    gx, gy = (W + 15) // 16, (H + 15) // 16
    u = np.empty((Cn, N, 2), np.float32)
    r = np.empty((Cn, N, 2), np.int32)
    for c in range(Cn):
        k = rng.integers(0, 5, N)
        ext = np.array([W, H], np.float32)
        edge = rng.integers(0, 2, (N, 2)) * ext + rng.uniform(-20, 20, (N, 2))  # near a border
        inside = rng.uniform(-0.2, 1.2, (N, 2)) * ext
        tiles = rng.integers(-2, max(gx, gy) + 2, (N, 2)) * 16.0  # exactly on tile lines
        u[c] = np.where(k[:, None] < 2, edge, np.where(k[:, None] < 4, inside, tiles))
        r[c] = np.where(rng.random((N, 2)) < 0.1, 0, rng.integers(0, 40, (N, 2)))
        r[c, :50] = rng.integers(200, 5000, (50, 2))  # huge
    out = np.empty((Cn * N, 4), np.int32)
    us, ar = np.ascontiguousarray(u.reshape(-1, 2)), np.ascontiguousarray(r.reshape(-1, 2))
    rect_shim.tile_rects(Cn * N, N, 1, us.ctypes.data_as(C.c_void_p), ar.ctypes.data_as(C.c_void_p), gx, gy,
                         out.ctypes.data_as(C.c_void_p))
    out = out.reshape(Cn, N, 4)
    for c in range(Cn):
        want = _single_rect_model(u[c], r[c], gx, gy)
        want[:, 2:] += c * gy
        np.testing.assert_array_equal(out[c], want)
        assert (out[c, :, 2:] >= c * gy).all() and (out[c, :, 2:] <= (c + 1) * gy).all()
    # the single frame's form is the batch's camera 0
    one = np.empty((N, 4), np.int32)
    rect_shim.tile_rects(N, N, 0, np.ascontiguousarray(u[0]).ctypes.data_as(C.c_void_p),
                         np.ascontiguousarray(r[0]).ctypes.data_as(C.c_void_p), gx, gy, one.ctypes.data_as(C.c_void_p))
    np.testing.assert_array_equal(one, out[0])
