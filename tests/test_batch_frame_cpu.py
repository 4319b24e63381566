"""The argument errors of the batch entry points (gsb_splat_{bin,render,forward,backward}_batch and
their RGB-D forms, gsb_preprocess_{forward,backward}_batch and _batch_pose): each call fails one
named check and must answer -1 with exactly that check's text.  Also the checks the one-camera and
the batch frames share since they run through one frame core: 2^30 patches or more in render and
backward, and the tile grid of the colour backward, refused on both paths.  The calls run in a
child process that sees no CUDA device, so a call that wrongly gets past its checks fails with a
CUDA error instead of reaching a GPU."""
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# as in test_splat_frame_cpu: any 256-byte aligned address stands for a device buffer
PTR = 0x10000000
MIS16, MIS8 = PTR + 8, PTR + 4
WIDE = 16 * 65536  # a width of 65536 tiles
BIG = 1 << 40
P30 = 1 << 30
RADIAL = "radial"  # intrinsics rows with radial coefficients (host memory)

CASES = [
    # binning
    ("gsb_splat_bin_batch", {"C": 0}, "splat_bin_batch: C < 1"),
    ("gsb_splat_bin_batch", {"C": -1}, "splat_bin_batch: C < 1"),
    ("gsb_splat_bin_batch", {"H": 0}, "splat_bin_batch: bad N/H/W"),
    ("gsb_splat_bin_batch", {"N": -1}, "splat_bin_batch: bad N/H/W"),
    ("gsb_splat_bin_batch", {"C": 2, "N": P30}, "splat_bin_batch: C N >= 2^31 records"),
    ("gsb_splat_bin_batch", {"W": WIDE}, "splat_bin_batch: more than 65535 tiles in a row or in the C frames' column"),
    ("gsb_splat_bin_batch", {"C": 3, "H": 16 * 21846},
     "splat_bin_batch: more than 65535 tiles in a row or in the C frames' column"),
    ("gsb_splat_bin_batch", {"bin_ws": MIS16}, "splat_bin_batch: bin_ws misaligned"),
    ("gsb_splat_bin_batch", {"bin_ws_bytes": 64}, "splat_bin_batch: bin workspace too small"),
    ("gsb_splat_bin_batch", {"bin_ws": None}, "splat_bin_batch: null workspace / P_host"),
    ("gsb_splat_bin_batch", {"P_host": None}, "splat_bin_batch: null workspace / P_host"),
    ("gsb_splat_bin_batch", {"areas": None}, "splat_bin_batch: null pointer"),
    # render
    ("gsb_splat_render_batch", {"C": 0}, "splat_batch: C < 1"),
    ("gsb_splat_render_batch", {"W": -1}, "splat_batch: bad N/H/W"),
    ("gsb_splat_render_batch", {"C": 64, "N": 1 << 25}, "splat_batch: C N >= 2^31 records"),
    ("gsb_splat_render_batch", {"C": 1 << 21}, "splat_batch: more than 65535 tiles in a row or in the C frames' column"),
    ("gsb_splat_render_batch", {"bin_ws": MIS16}, "splat_batch: bin_ws misaligned"),
    ("gsb_splat_render_batch", {"P": -1}, "splat_batch: bad P"),
    ("gsb_splat_render_batch", {"P": P30}, "splat_batch: more than 2^30 patches"),
    ("gsb_splat_render_batch", {"colors": None}, "splat_batch: null pointer"),
    ("gsb_splat_render_batch", {"gsid_per_patch": None}, "splat_batch: null pointer"),
    ("gsb_splat_render_batch", {"image": None}, "splat_batch: null output"),
    ("gsb_splat_render_batch", {"final_tau": MIS16}, "splat_batch: misaligned output"),
    ("gsb_splat_render_batch", {"patch_range_per_tile": MIS8}, "splat_batch: misaligned output"),
    ("gsb_splat_render_batch", {"packed_records": MIS16}, "splat: packed_records misaligned"),
    ("gsb_splat_render_batch", {"ws": MIS16}, "splat_batch: ws misaligned"),
    ("gsb_splat_render_batch", {"ws_bytes": 64}, "splat_batch: workspace too small"),
    ("gsb_splat_render_batch_rgbd", {"alpha_image": None}, "splat_batch_rgbd: null depth_image / alpha_image"),
    ("gsb_splat_render_batch_rgbd", {"C": 0}, "splat_batch_rgbd: C < 1"),
    ("gsb_splat_render_batch_rgbd", {"P": P30}, "splat_batch_rgbd: more than 2^30 patches"),
    ("gsb_splat_render_batch_rgbd", {"depth_image": MIS16}, "splat: misaligned depth_image / alpha_image"),
    ("gsb_splat_render_batch_rgbd", {"contrib": None}, "splat_batch_rgbd: null output"),
    ("gsb_splat_render_batch_rgbd", {"ws_bytes": 64}, "splat_batch_rgbd: workspace too small"),
    # the capacity path (the checks made before its status event is created)
    ("gsb_splat_forward_batch", {"C": 0}, "splat_batch: C < 1"),
    ("gsb_splat_forward_batch", {"H": 0}, "splat_batch: bad N/H/W"),
    ("gsb_splat_forward_batch", {"C": 2, "N": P30}, "splat_batch: C N >= 2^31 records"),
    ("gsb_splat_forward_batch", {"W": WIDE}, "splat_batch: more than 65535 tiles in a row or in the C frames' column"),
    ("gsb_splat_forward_batch", {"bin_ws": MIS16}, "splat_batch: bin_ws misaligned"),
    ("gsb_splat_forward_batch", {"bin_ws_bytes": 64}, "splat_batch: bin workspace too small"),
    ("gsb_splat_forward_batch", {"P_cap": 0}, "splat_batch: bad P_cap (2^30 patches or more)"),
    ("gsb_splat_forward_batch", {"P_cap": P30}, "splat_batch: bad P_cap (2^30 patches or more)"),
    ("gsb_splat_forward_batch", {"status_host": None}, "splat_batch: null pointer"),
    ("gsb_splat_forward_batch", {"areas": None}, "splat_batch: null pointer"),
    ("gsb_splat_forward_batch_rgbd", {"depth_image": None}, "splat_batch_rgbd: null depth_image / alpha_image"),
    ("gsb_splat_forward_batch_rgbd", {"C": -3}, "splat_batch_rgbd: C < 1"),
    ("gsb_splat_forward_batch_rgbd", {"P_cap": -5}, "splat_batch_rgbd: bad P_cap (2^30 patches or more)"),
    ("gsb_splat_forward_batch_rgbd", {"gsid_per_patch": None}, "splat_batch_rgbd: null pointer"),
    # backward
    ("gsb_splat_backward_batch", {"C": 0}, "splatB_batch: C < 1"),
    ("gsb_splat_backward_batch", {"N": -1}, "splatB_batch: bad N/H/W"),
    ("gsb_splat_backward_batch", {"C": 2, "N": P30}, "splatB_batch: C N >= 2^31 records"),
    ("gsb_splat_backward_batch", {"C": 3, "H": 16 * 21846},
     "splatB_batch: more than 65535 tiles in a row or in the C frames' column"),
    ("gsb_splat_backward_batch", {"P": -1}, "splatB_batch: bad P"),
    ("gsb_splat_backward_batch", {"P": P30}, "splatB_batch: more than 2^30 patches"),
    ("gsb_splat_backward_batch", {"moments_out": None}, "splatB_batch: null pointer"),
    ("gsb_splat_backward_batch", {"ws": None}, "splatB_batch: null pointer"),
    ("gsb_splat_backward_batch", {"ws_bytes": 64}, "splatB_batch: workspace too small"),
    ("gsb_splat_backward_batch", {"dloss_dgammas": None}, "splatB_batch: null pointer"),
    ("gsb_splat_backward_batch", {"packed_records": MIS16}, "splatB_batch: packed_records misaligned"),
    ("gsb_splat_backward_batch_rgbd", {"C": 0}, "splatB_batch_rgbd: C < 1"),
    ("gsb_splat_backward_batch_rgbd", {"P": P30}, "splatB_batch_rgbd: more than 2^30 patches"),
    ("gsb_splat_backward_batch_rgbd", {"dloss_ddepths": None}, "splatB_batch_rgbd: null pointer"),
    ("gsb_splat_backward_batch_rgbd", {"dloss_ddepths": None, "P": 0}, "splatB_batch_rgbd: null pointer"),
    ("gsb_splat_backward_batch_rgbd", {"dloss_dalpha_image": None}, "splatB_batch_rgbd: null pointer"),
    ("gsb_splat_backward_batch_rgbd", {"depths": None}, "splatB_batch_rgbd: null pointer"),
    ("gsb_splat_backward_batch_rgbd", {"ws_bytes": 64}, "splatB_batch_rgbd: workspace too small"),
    # the per-Gaussian entry points
    ("gsb_preprocess_forward_batch", {"C": 0}, "preprocess_batch: C < 1"),
    ("gsb_preprocess_forward_batch", {"C": 65}, "preprocess_batch: C > GSB_BATCH_MAX_CAMERAS"),
    ("gsb_preprocess_forward_batch", {"N": -1}, "preprocess_batch: N < 0"),
    ("gsb_preprocess_forward_batch", {"N": P30}, "preprocess_batch: C N >= 2^31 records"),
    ("gsb_preprocess_forward_batch", {"sh_dim3": 2}, "preprocess_batch: shs.shape[1]/3 must be 1, 4, 9 or 16"),
    ("gsb_preprocess_forward_batch", {"intrinsics": None}, "preprocess_batch: null intrinsics"),
    ("gsb_preprocess_forward_batch", {"intrinsics": RADIAL},
     "preprocess_batch: radial coefficients are for the fisheye and opencv models only"),
    ("gsb_preprocess_forward_batch", {"camera_model": 5}, "preprocess_batch: unknown camera model"),
    ("gsb_preprocess_forward_batch", {"width": 0.0, "camera_model": 4},
     "preprocess_batch: the opencv model needs width and height > 0"),
    ("gsb_preprocess_forward_batch", {"records": MIS16}, "preprocess_batch: records misaligned"),
    ("gsb_preprocess_forward_batch", {"poses": None}, "preprocess_batch: null pointer"),
    ("gsb_preprocess_forward_batch", {"areas": None}, "preprocess_batch: null pointer"),
    ("gsb_preprocess_backward_batch", {"C": 0}, "preprocessB_batch: C < 1"),
    ("gsb_preprocess_backward_batch", {"C": 65}, "preprocessB_batch: C > GSB_BATCH_MAX_CAMERAS"),
    ("gsb_preprocess_backward_batch", {"N": -1}, "preprocessB_batch: N < 0"),
    ("gsb_preprocess_backward_batch", {"sh_dim3": 0}, "preprocessB_batch: shs.shape[1]/3 must be 1, 4, 9 or 16"),
    ("gsb_preprocess_backward_batch", {"intrinsics": None}, "preprocessB_batch: null intrinsics"),
    ("gsb_preprocess_backward_batch", {"camera_model": -1}, "preprocessB_batch: unknown camera model"),
    ("gsb_preprocess_backward_batch", {"shs": None}, "preprocessB_batch: null pointer"),
    ("gsb_preprocess_backward_batch", {"cinv2ds": None}, "preprocessB_batch: null pointer"),
    ("gsb_preprocess_backward_batch", {"dloss_dalphas_out": None}, "preprocessB_batch: null output"),
    ("gsb_preprocess_backward_batch_pose", {"C": 0}, "preprocessB_batch_pose: C < 1"),
    ("gsb_preprocess_backward_batch_pose", {"N": P30}, "preprocessB_batch_pose: C N >= 2^31 records"),
    ("gsb_preprocess_backward_batch_pose", {"camera_model": 3}, "preprocessB_batch_pose: unknown camera model"),
    ("gsb_preprocess_backward_batch_pose", {"moments": None}, "preprocessB_batch_pose: null pointer"),
    ("gsb_preprocess_backward_batch_pose", {"dloss_dpws": None},
     "preprocessB_batch_pose: per-Gaussian outputs must be all set or all null"),
    ("gsb_preprocess_backward_batch_pose", {"dloss_dposes": None}, "preprocessB_batch_pose: null dloss_dposes"),
    ("gsb_preprocess_backward_batch_pose", {"ws": MIS16}, "preprocessB_batch_pose: workspace misaligned"),
    ("gsb_preprocess_backward_batch_pose", {"ws": None}, "preprocessB_batch_pose: workspace too small"),
    ("gsb_preprocess_backward_batch_pose", {"ws_bytes": 64}, "preprocessB_batch_pose: workspace too small"),
    # refused on both paths: 2^30 patches or more, and the colour backward's tile grid
    ("gsb_splat_render", {"P": P30}, "splat: more than 2^30 patches"),
    ("gsb_splat_render_rgbd", {"P": P30}, "splat: more than 2^30 patches"),
    ("gsb_splat_backward", {"P": P30}, "splatB: more than 2^30 patches"),
    ("gsb_splat_backward", {"W": WIDE}, "splatB: more than 65535 tiles in a row or column"),
    ("gsb_splat_backward_rgbd", {"P": P30}, "splatB: more than 2^30 patches"),
    ("gsb_splat_backward_rgbd", {"H": WIDE}, "splatB: more than 65535 tiles in a row or column"),
    ("gsb_splat_backward_abs", {"P": P30}, "splatB: more than 2^30 patches"),
    ("gsb_splat_backward_abs", {"W": WIDE}, "splatB: more than 65535 tiles in a row or column"),
    ("gsb_splat_backward_rgbd_abs", {"P": P30}, "splatB: more than 2^30 patches"),
    ("gsb_splat_backward_rgbd_abs", {"W": WIDE}, "splatB: more than 65535 tiles in a row or column"),
    ("gsb_splat_backward_batch", {"W": WIDE}, "splatB_batch: more than 65535 tiles in a row or in the C frames' column"),
]


def _param_names():
    """entry point -> its parameter names, from the header's declarations"""
    with open(os.path.join(ROOT, "include", "gsplat_b200.h")) as f:
        src = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    return {m.group(1): [re.findall(r"\w+", p)[-1] for p in m.group(2).split(",")]
            for m in re.finditer(r"\bint\s+(gsb_\w+)\s*\(([^;]*)\)\s*;", src)}


def _run_cases():
    """(rc, gsb_last_error) of every case, in a process without a CUDA device"""
    import ctypes as C
    from easygaussiansplatting_b200 import _lib
    lib = _lib.load()
    names = _param_names()
    # written or read on the host: real buffers
    status, P_host, dk = (C.c_uint32 * 4)(), C.c_int64(), C.c_uint32()
    rows = (C.c_float * (8 * 65))(*([200.0, 200.0, 32.0, 32.0, 0, 0, 0, 0] * 65))
    radial = (C.c_float * (8 * 2))(*([200.0, 200.0, 32.0, 32.0, 0.1, 0, 0, 0] * 2))
    base = {"C": 2, "H": 64, "W": 64, "N": 10, "P": 100, "P_cap": 1000, "depth_key_max": 255, "depth_key_cap": 255,
            "ws_bytes": BIG, "bin_ws_bytes": BIG, "status_host": C.addressof(status), "stream": None,
            "P_host": C.pointer(P_host), "depth_key_max_host": C.pointer(dk), "sh_dim3": 16, "camera_model": 0,
            "width": 64.0, "height": 64.0, "intrinsics": C.addressof(rows)}
    out = []
    for entry, broken, _ in CASES:
        args = {n: base.get(n, PTR) for n in names[entry]}
        assert set(broken) <= set(args), (entry, broken)
        args.update(broken)
        if args.get("intrinsics") == RADIAL:
            args["intrinsics"] = C.addressof(radial)
        rc = getattr(lib, entry)(*args.values())
        out.append((rc, lib.gsb_last_error().decode()))
    return out


def test_batch_entry_points_name_the_failed_check():
    from easygaussiansplatting_b200 import build
    build.build()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.abspath(__file__)], capture_output=True, text=True, env=env,
                       cwd=ROOT, timeout=300)
    assert r.returncode == 0, r.stderr[-4000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(got) == len(CASES)
    bad = [(entry, broken, want, tuple(g)) for (entry, broken, want), g in zip(CASES, got)
           if tuple(g) != (-1, "argument error: " + want)]
    assert not bad, "\n".join(map(str, bad))


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    print(json.dumps(_run_cases()))
