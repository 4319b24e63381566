"""The batch's camera gradients without a GPU (DESIGN 3.22): the workspace query, every argument error of
gsb_preprocess_backward_batch_pose returned before any launch, the Python argument rules, and the new
kernels in the sm_90a cubin without stack or spills."""
import ctypes as C
import os
import re
import subprocess

import pytest
import torch

from easygaussiansplatting_b200 import _lib, build, ops
from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFusedBatchPose

CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def _err(lib):
    return lib.gsb_last_error().decode()


def test_workspace_query(lib):
    q = lib.gsb_preprocess_backward_batch_pose_workspace_bytes
    for Cn, N in ((1, 1), (1, 128), (1, 129), (3, 1000), (8, 2_000_000), (64, 1 << 24), (2, 0)):
        assert q(Cn, N) == Cn * ((N + 127) // 128) * 64, (Cn, N)
        assert q(Cn, N) == Cn * lib.gsb_preprocess_backward_pose_workspace_bytes(N)
    # what the entry point refuses sizes nothing (no int overflow of C N)
    for Cn, N in ((0, 1000), (-1, 1000), (2, 1 << 30), (64, 1 << 26), (1, -1)):
        assert q(Cn, N) == 0, (Cn, N)


def _call(lib, Cn=2, N=10, k3=16, intr=None, model=0, ins=True, outs=None, dposes=True, ws=None, ws_bytes=None,
          buf=None):
    """gsb_preprocess_backward_batch_pose with fake (never dereferenced) device pointers"""
    fake = buf + 64  # 16-byte aligned host address: nothing may be launched on it
    base = [fake] * 5 if ins else [None] * 5  # pws, rots, scales, shs, poses
    up = [fake, fake] if ins else [None, None]  # moments, cinv2ds
    outs = [fake] * 6 if outs is None else outs
    need = lib.gsb_preprocess_backward_batch_pose_workspace_bytes(Cn, N)
    return lib.gsb_preprocess_backward_batch_pose(
        Cn, N, k3, *base, intr, model, 16.0, 16.0, *up, None, None, *outs, fake if dposes else None,
        buf if ws is None else ws, need if ws_bytes is None else ws_bytes, None)


def test_argument_errors_before_any_launch(lib):
    store = (C.c_char * 4096)()
    buf = C.addressof(store) + (-C.addressof(store)) % 16
    rows = (C.c_float * 16)(200.0, 200.0, 8.0, 8.0, 0, 0, 0, 0, -1.0, 200.0, 8.0, 8.0, 0, 0, 0, 0)
    bad_intr = C.addressof(rows)  # camera 1: fx < 0
    ok_rows = (C.c_float * 16)(200.0, 200.0, 8.0, 8.0, 0, 0, 0, 0, 210.0, 205.0, 8.0, 8.0, 0, 0, 0, 0)
    intr = C.addressof(ok_rows)
    idx = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())].index(
        "preprocess_backward_batch")
    before = lib.gsb_profile_launches(idx), lib.gsb_profile_launches(-1)
    f = buf + 64
    cases = [
        # everything gsb_preprocess_backward_batch refuses
        (dict(Cn=0), "C < 1"),
        (dict(Cn=65, intr=intr), "GSB_BATCH_MAX_CAMERAS"),
        (dict(N=-1, intr=intr), "N < 0"),
        (dict(Cn=2, N=1 << 30, intr=intr), "2^31"),
        (dict(k3=5, intr=intr), "shs.shape[1]/3"),
        (dict(intr=None), "null intrinsics"),
        (dict(intr=bad_intr, model=2), "fx and fy must be > 0"),
        (dict(intr=intr, model=7), "unknown camera model"),
        (dict(intr=intr, ins=False), "null pointer"),
        # a mix of NULL and set per-Gaussian outputs
        (dict(intr=intr, outs=[None, f, f, f, f, f]), "all set or all null"),
        (dict(intr=intr, outs=[f, f, f, f, f, None]), "all set or all null"),
        (dict(intr=intr, outs=[None, None, None, None, f, None]), "all set or all null"),
        # the camera gradients' output and workspace
        (dict(intr=intr, dposes=False), "null dloss_dposes"),
        (dict(intr=intr, ws=buf + 4), "misaligned"),
        (dict(intr=intr, ws_bytes=63), "too small"),
        (dict(intr=intr, N=1000, ws_bytes=7 * 64), "too small"),
        (dict(intr=intr, ws=0), "too small"),
    ]
    for kw, msg in cases:
        if kw.get("ws") == 0:
            kw["ws"] = None
            rc = lib.gsb_preprocess_backward_batch_pose(2, 10, 16, *([f] * 5), intr, 0, 16.0, 16.0, f, f, None, None,
                                                        *([f] * 6), f, None, 128, None)
        else:
            rc = _call(lib, buf=buf, **kw)
        assert rc != 0 and msg in _err(lib), (kw, msg, _err(lib))
    assert (lib.gsb_profile_launches(idx), lib.gsb_profile_launches(-1)) == before


def test_python_argument_rules():
    R, t = torch.eye(3), torch.zeros(3)
    cams = [Camera(64, 48, 50.0, 50.0, 32.0, 24.0, R, t), Camera(64, 48, 55.0, 52.0, 31.0, 25.0, R, t)]
    poses = torch.arange(30, dtype=torch.float32).reshape(2, 15)
    bc = ops.BatchCameras(cams, "cpu", poses=poses)
    assert torch.equal(bc.poses, poses) and bc.intrinsics[1, :4].tolist() == [55.0, 52.0, 31.0, 25.0]
    own = ops.BatchCameras(cams, "cpu")
    assert torch.equal(own.poses[0, :9], R.reshape(-1)) and torch.equal(own.poses[1, 9:12], t)
    for bad in (torch.zeros(3, 15), torch.zeros(2, 12), torch.zeros(2, 15, dtype=torch.float64), [[0.0] * 15] * 2):
        with pytest.raises(ValueError, match="poses"):
            ops.BatchCameras(cams, "cpu", poses=bad)
    z = torch.zeros(0)
    with pytest.raises(ValueError, match="pose_only"):
        ops.preprocessB_batch(z, z, z, z, cams, z, z, pose_only=True)
    N = 5
    g = [torch.zeros(N, 3), torch.zeros(N, 48), torch.zeros(N, 1), torch.zeros(N, 3), torch.zeros(N, 4),
         torch.zeros(2, N, 2)]
    for Rs, ts, ws in ((torch.zeros(3, 3, 3), torch.zeros(2, 3), torch.zeros(2, 3)),
                       (torch.zeros(2, 3, 3), torch.zeros(2, 4), torch.zeros(2, 3)),
                       (torch.zeros(2, 3, 3), torch.zeros(2, 3), None)):
        with pytest.raises(ValueError, match="Rcws|tcws|twcs"):
            GSFunctionFusedBatchPose.apply(*g, Rs, ts, ws, cams)


def _res_usage(so):
    out = subprocess.run([CUOBJDUMP, "-res-usage", so], capture_output=True, text=True, check=True).stdout
    res, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", line)
        if m and name:
            res[name] = tuple(int(x) for x in m.groups())
            name = None
    return res


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not installed")
def test_new_kernels_in_the_cubin_without_stack_or_spills(lib):
    res = _res_usage(_lib.LIB_PATH)
    pose = {k: v for k, v in res.items() if "k_preprocess_bwd_batch_pose" in k}
    # every K3 (1, 4, 9, 16) x DEPTH x AA x camera model (4)
    assert len(pose) == 64, sorted(pose)
    red = [k for k in res if "k_pose_reduce_batch" in k]
    assert len(red) == 1
    for k in list(pose) + red:
        reg, stack, shared, local = res[k]
        assert stack == 0 and local == 0, (k, res[k])
        assert reg <= 128, (k, res[k])  # room for 4 CTAs of 128 threads per SM
