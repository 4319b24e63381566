"""Batched 2D Gaussian Splatting (DESIGN 3.25) without a GPU: every argument error of the
gsb_2dgs_batch_* entry points (answered before any launch, in a process that sees no CUDA device),
the Python classes' refusals, the ctypes declarations against the header, the profile ids, and
loss.depth_to_normal on a batch of depth maps against single calls."""
import json
import os
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PTR = 0x10000000
MIS16 = PTR + 8
MIS4 = PTR + 2
BIG = 1 << 40
TALL = 16 * 21846  # 3 frames of 21846 tile rows: one row more than the tall frame takes

FWD = "gsb_2dgs_batch_preprocess_forward"
BWD = "gsb_2dgs_batch_preprocess_backward"
CASES = [
    (FWD, {"C": 0}, "2dgs_batch_preprocess: C < 1"),
    (FWD, {"C": 65}, "2dgs_batch_preprocess: C > GSB_BATCH_MAX_CAMERAS"),
    (FWD, {"N": 1 << 30}, "2dgs_batch_preprocess: C N >= 2^31 records"),
    (FWD, {"camera_model": 1}, "2dgs_batch_preprocess: pinhole cameras only"),
    (FWD, {"camera_model": 3}, "2dgs_batch_preprocess: pinhole cameras only"),
    (FWD, {"sh_dim3": 2}, "2dgs_batch_preprocess: shs.shape[1]/3 must be 1, 4, 9 or 16"),
    (FWD, {"intrinsics": None}, "2dgs_batch_preprocess: null intrinsics"),
    (FWD, {"records": MIS16}, "2dgs_batch_preprocess: records misaligned"),
    (FWD, {"poses": None}, "2dgs_batch_preprocess: null pointer"),
    (FWD, {"colors": None}, "2dgs_batch_preprocess: null pointer"),
    (BWD, {"C": -1}, "2dgs_batch_preprocessB: C < 1"),
    (BWD, {"C": 65}, "2dgs_batch_preprocessB: C > GSB_BATCH_MAX_CAMERAS"),
    (BWD, {"camera_model": 2}, "2dgs_batch_preprocessB: pinhole cameras only"),
    (BWD, {"rows": None}, "2dgs_batch_preprocessB: null pointer"),
    ("gsb_2dgs_batch_render", {"C": 0}, "2dgs_batch: C < 1"),
    ("gsb_2dgs_batch_render", {"C": 65}, "2dgs_batch: C > GSB_BATCH_MAX_CAMERAS"),
    ("gsb_2dgs_batch_render", {"C": 2, "N": 1 << 30}, "2dgs_batch: C N >= 2^31 records"),
    ("gsb_2dgs_batch_render", {"H": TALL}, "2dgs_batch: more than 65535 tiles in a row or in the C frames' column"),
    ("gsb_2dgs_batch_render", {"P": 1 << 30}, "2dgs_batch: more than 2^30 patches"),
    ("gsb_2dgs_batch_render", {"P": -1}, "2dgs_batch: bad P"),
    ("gsb_2dgs_batch_render", {"records": None}, "2dgs_batch: null pointer"),
    ("gsb_2dgs_batch_render", {"image": MIS16}, "2dgs_batch: misaligned output"),
    ("gsb_2dgs_batch_render", {"normal_image": MIS16}, "splat_surfel: misaligned output"),
    ("gsb_2dgs_batch_render", {"records": MIS16}, "splat_surfel: records misaligned"),
    ("gsb_2dgs_batch_render", {"ws_bytes": 64}, "2dgs_batch: workspace too small"),
    ("gsb_2dgs_batch_forward", {"C": 0}, "2dgs_batch: C < 1"),
    ("gsb_2dgs_batch_forward", {"H": TALL}, "2dgs_batch: more than 65535 tiles in a row or in the C frames' column"),
    ("gsb_2dgs_batch_forward", {"P_cap": 1 << 30}, "2dgs_batch: bad P_cap (2^30 patches or more)"),
    ("gsb_2dgs_batch_forward", {"bin_ws": MIS16}, "2dgs_batch: bin_ws misaligned"),
    ("gsb_2dgs_batch_forward", {"bin_ws_bytes": 64}, "2dgs_batch: bin workspace too small"),
    ("gsb_2dgs_batch_forward", {"status_host": None}, "2dgs_batch: null pointer"),
    ("gsb_2dgs_batch_backward", {"C": 65}, "2dgs_batchB: C > GSB_BATCH_MAX_CAMERAS"),
    ("gsb_2dgs_batch_backward", {"H": TALL}, "2dgs_batchB: more than 65535 tiles in a row or in the C frames' column"),
    ("gsb_2dgs_batch_backward", {"P": 1 << 30}, "2dgs_batchB: more than 2^30 patches"),
    ("gsb_2dgs_batch_backward", {"rows": None}, "2dgs_batchB: null output"),
    ("gsb_2dgs_batch_backward", {"ws_bytes": 64}, "2dgs_batchB: workspace too small"),
    ("gsb_2dgs_batch_backward", {"records": MIS16}, "2dgs_batchB: misaligned input"),
    ("gsb_2dgs_batch_render_geometry", {"near": 0.0}, "2dgs_batch: near <= 0"),
    ("gsb_2dgs_batch_render_geometry", {"moments": MIS16}, "2dgs_batch: misaligned geometry plane"),
    ("gsb_2dgs_batch_render_geometry", {"C": 65}, "2dgs_batch: C > GSB_BATCH_MAX_CAMERAS"),
    ("gsb_2dgs_batch_forward_geometry", {"distortion": None}, "2dgs_batch: null geometry plane"),
    ("gsb_2dgs_batch_forward_geometry", {"H": TALL}, "2dgs_batch: more than 65535 tiles in a row or in the C frames' column"),
    ("gsb_2dgs_batch_backward_geometry", {"far": 0.1}, "2dgs_batchB: far <= near"),
    ("gsb_2dgs_batch_backward_geometry", {"moments": None}, "2dgs_batchB: null geometry plane"),
    ("gsb_2dgs_batch_backward_geometry", {"median_contrib": MIS4}, "2dgs_batchB: misaligned geometry plane"),
    ("gsb_2dgs_batch_backward_geometry", {"C": 0}, "2dgs_batchB: C < 1"),
]


def _decls():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "gsplat_b200.h")).read(), flags=re.S)
    return {m.group(1): m.group(2) for m in re.finditer(r"\b(gsb_2dgs_batch_\w+)\s*\(([^;]*)\)\s*;", src)}


def _run_cases():
    import ctypes as C
    from easygaussiansplatting_b200 import _lib
    lib = _lib.load()
    names = {k: [re.findall(r"\w+", p)[-1] for p in v.split(",")] for k, v in _decls().items()}
    status = (C.c_uint32 * 4)()
    rows = (C.c_float * (8 * 65))(*([200.0, 200.0, 32.0, 32.0, 0, 0, 0, 0] * 65))
    base = {"C": 3, "H": 64, "W": 64, "N": 10, "P": 100, "P_cap": 1000, "depth_key_max": 255, "depth_key_cap": 255,
            "ws_bytes": BIG, "bin_ws_bytes": BIG, "status_host": C.addressof(status), "stream": None,
            "sh_dim3": 16, "camera_model": 0, "width": 64.0, "height": 64.0, "intrinsics": C.addressof(rows),
            "near": 0.2, "far": 100.0}
    out = []
    for entry, broken, _ in CASES:
        args = {n: base.get(n, PTR) for n in names[entry]}
        assert set(broken) <= set(args), (entry, broken)
        args.update(broken)
        rc = getattr(lib, entry)(*args.values())
        out.append((rc, lib.gsb_last_error().decode()))
    return out


def test_entry_points_refuse_before_any_launch():
    from easygaussiansplatting_b200 import build
    build.build()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.abspath(__file__)], capture_output=True, text=True, env=env, cwd=ROOT,
                       timeout=300)
    assert r.returncode == 0, r.stderr[-4000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    bad = [(e, b, want, tuple(g)) for (e, b, want), g in zip(CASES, got) if tuple(g) != (-1, "argument error: " + want)]
    assert len(got) == len(CASES) and not bad, "\n".join(map(str, bad))


def test_declarations_workspace_and_profile_ids():
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    lib = _lib.load()
    decls = _decls()
    assert sorted(decls) == sorted("gsb_2dgs_batch_" + s for s in (
        "workspace_bytes", "preprocess_forward", "preprocess_backward", "render", "forward", "backward",
        "render_geometry", "forward_geometry", "backward_geometry"))
    syms = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    for name, args in decls.items():
        assert len(_lib.SIGNATURES[name][1]) == len(args.split(",")), name
        assert re.search(r"\bT %s$" % name, syms, re.M), name
    assert lib.gsb_abi_version() == 1
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    i = names.index("rects+scan_batch")  # just before the 3DGS batch's ids
    assert names[i - 6:i] == ["surfel_forward_batch", "draw_surfel_batch", "draw_surfel_backward_batch",
                          "surfel_backward_batch", "draw_2dgs_batch", "draw_2dgs_backward_batch"]
    # the workspace is the tall frame's sort layout; 0 for what the entry points refuse
    ws = lib.gsb_2dgs_batch_workspace_bytes
    assert ws(4, 1000, 64, 64, 0) == lib.gsb_splat_batch_workspace_bytes(4, 1000, 64, 64, 0) > 0
    assert ws(4, 1000, 64, 64, 100000) > ws(4, 1000, 64, 64, 0)
    assert ws(0, 10, 64, 64, 0) == 0 and ws(65, 10, 64, 64, 0) == 0 and ws(2, 1 << 30, 64, 64, 0) == 0


def test_batched_kernels_sm90a_no_local_memory():
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    res = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True).stdout
    found = dict(re.findall(r"Function (_ZN3gsb\d+k_(?:disk_\w+|draw_disk\w+|draw_2dgs\w*_batch)\S*):\s*\n\s*(REG:.*)",
                            res))
    kinds = sorted(set(re.sub(r"^_ZN3gsb\d+(k_[a-z0-9_]+).*$", r"\1", f) for f in found))
    assert kinds == ["k_disk_bwd_batch", "k_disk_fwd_batch", "k_draw_2dgs_batch", "k_draw_2dgs_bwd_batch",
                     "k_draw_disk_batch", "k_draw_disk_bwd_batch"], kinds
    assert len(found) == 12
    for f, r in found.items():
        assert "STACK:0" in r and "LOCAL:0" in r, (f, r)
        if "k_draw" in f:  # 4 CTAs of 128 threads per SM
            assert int(re.search(r"REG:(\d+)", r).group(1)) <= 128, (f, r)


def _cam(W=32, H=24, **kw):
    from easygaussiansplatting_b200.gsfunction import Camera
    return Camera(W, H, 20.0, 21.0, 16.0, 12.0, torch.eye(3), torch.zeros(3), **kw)


@pytest.mark.parametrize("cls", ["GSFunctionSurfelBatch", "GSFunctionSurfelGeometryBatch"])
def test_python_refusals(cls):
    from easygaussiansplatting_b200 import gsfunction
    fn = getattr(gsfunction, cls)
    N = 5
    a = (torch.zeros(N, 3), torch.zeros(N, 3), torch.zeros(N, 1), torch.zeros(N, 3), torch.zeros(N, 4),
         torch.zeros(2, N, 2))
    for bad in (_cam(antialiased=True), _cam(camera_model="ortho"), _cam(camera_model="fisheye"), _cam(W=48)):
        with pytest.raises(ValueError):
            fn.apply(*a, [_cam(), bad])
    ge = _cam()
    ge.grad_exchange = object()
    with pytest.raises(ValueError, match="grad_exchange"):
        fn.apply(*a, [_cam(), ge])
    with pytest.raises(ValueError, match="1 to 64 cameras"):
        fn.apply(*a[:5], torch.zeros(65, N, 2), [_cam()] * 65)
    with pytest.raises(ValueError, match=r"\[C, N, 2\]"):
        fn.apply(*a[:5], torch.zeros(3, N, 2), [_cam(), _cam()])
    if cls == "GSFunctionSurfelBatch":
        with pytest.raises(ValueError, match="filter3d"):
            fn.apply(*a, [_cam(), _cam()], torch.zeros(N))
        with pytest.raises(ValueError, match="us_abs"):
            fn.apply(*a, [_cam(), _cam()], None, torch.zeros(2, N, 2))
    else:
        with pytest.raises(ValueError, match="near and far"):
            fn.apply(*a, [_cam(), _cam()], torch.zeros(1))


def test_ops_refuse_other_camera_models():
    from easygaussiansplatting_b200 import ops
    bc = ops.BatchCameras([_cam(camera_model="ortho")] * 2, "cpu")
    with pytest.raises(ValueError, match="pinhole"):
        ops._surfel_batch_cams(bc, "cpu")
    bc = ops.BatchCameras([_cam(antialiased=True)] * 2, "cpu")
    with pytest.raises(ValueError, match="pinhole"):
        ops._surfel_batch_cams(bc, "cpu")


def test_depth_to_normal_of_a_batch_is_the_single_calls():
    from easygaussiansplatting_b200.loss import depth_to_normal
    g = torch.Generator().manual_seed(0)
    C, H, W = 3, 17, 23
    depth = 2.0 + torch.rand((C, H, W), generator=g, dtype=torch.float64)
    depth[1, 5:9, 4:10] = 0.0
    cams = [_cam(W, H) for _ in range(C)]
    for c, cam in enumerate(cams):
        cam.fx, cam.cy = 20.0 + c, 11.0 - c
    out = depth_to_normal(depth, cams)
    assert out.shape == (C, 3, H, W)
    for c in range(C):
        assert torch.equal(out[c], depth_to_normal(depth[c], cams[c]))
    d = depth.clone().requires_grad_()
    depth_to_normal(d, cams).sum().backward()
    ones = torch.ones(3, H, W, dtype=depth.dtype)
    want = torch.stack([torch.autograd.functional.vjp(lambda z, c=c: depth_to_normal(z, cams[c]), depth[c], ones)[1]
                        for c in range(C)])
    assert torch.allclose(d.grad, want, atol=1e-12)
    with pytest.raises(ValueError):
        depth_to_normal(depth, cams[:2])
    with pytest.raises(ValueError):
        depth_to_normal(depth[0], cams)


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    print(json.dumps(_run_cases()))
