"""The argument errors of the frame entry points (gsb_splat_render / _forward / _backward and their
RGB-D, AbsGS and surfel forms): each call fails one named check and must answer -1 with exactly
that check's text.  The calls run in a child process that sees no CUDA device, so a call that
wrongly gets past its checks fails with a CUDA error instead of reaching a GPU."""
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Device pointers are never dereferenced on the host: any 256-byte aligned address stands for a
# buffer, and +8 / +4 break the 16-byte (planes, records, workspaces) and 8-byte (tile ranges)
# alignment the entry points require.
PTR = 0x10000000
MIS16, MIS8 = PTR + 8, PTR + 4
WIDE = 16 * 65536  # a width of 65536 tiles
BIG = 1 << 40      # workspace sizes that always suffice

# (entry point, {parameter: value} that breaks one check, the error text after "argument error: ")
CASES = [
    # the exact colour frame
    ("gsb_splat_render", {"H": 0}, "splat: bad N/H/W"),
    ("gsb_splat_render", {"N": -1}, "splat: bad N/H/W"),
    ("gsb_splat_render", {"W": WIDE}, "splat: more than 65535 tiles in a row or column"),
    ("gsb_splat_render", {"bin_ws": MIS16}, "splat: bin_ws misaligned"),
    ("gsb_splat_render", {"P": -1}, "splat: bad P"),
    ("gsb_splat_render", {"colors": None}, "splat: null pointer"),
    ("gsb_splat_render", {"image": None}, "splat: null output"),
    ("gsb_splat_render", {"patch_range_per_tile": None}, "splat: null output"),
    ("gsb_splat_render", {"final_tau": MIS16}, "splat: misaligned output"),
    ("gsb_splat_render", {"patch_range_per_tile": MIS8}, "splat: misaligned output"),
    ("gsb_splat_render", {"packed_records": MIS16}, "splat: packed_records misaligned"),
    ("gsb_splat_render", {"ws": MIS16}, "splat: ws misaligned"),
    ("gsb_splat_render", {"ws_bytes": 64}, "splat: workspace too small"),
    ("gsb_splat_render_rgbd", {"W": WIDE}, "splat: more than 65535 tiles in a row or column"),
    ("gsb_splat_render_rgbd", {"alpha_image": None}, "splat_rgbd: null depth_image / alpha_image"),
    ("gsb_splat_render_rgbd", {"depth_image": MIS16}, "splat: misaligned depth_image / alpha_image"),
    ("gsb_splat_render_rgbd", {"contrib": None}, "splat: null output"),
    ("gsb_splat_render_rgbd", {"image": MIS16}, "splat: misaligned output"),
    ("gsb_splat_render_rgbd", {"ws_bytes": 64}, "splat: workspace too small"),
    # the colour frame on the capacity path (the checks made before its status event is created)
    ("gsb_splat_forward", {"W": -1}, "splat: bad N/H/W"),
    ("gsb_splat_forward", {"H": WIDE}, "splat: more than 65535 tiles in a row or column"),
    ("gsb_splat_forward", {"bin_ws": MIS16}, "splat: bin_ws misaligned"),
    ("gsb_splat_forward", {"bin_ws_bytes": 64}, "splat: bin workspace too small"),
    ("gsb_splat_forward", {"P_cap": 0}, "splat_forward: bad P_cap"),
    ("gsb_splat_forward", {"P_cap": 1 << 30}, "splat_forward: bad P_cap"),
    ("gsb_splat_forward", {"status_host": None}, "splat_forward: null pointer"),
    ("gsb_splat_forward", {"areas": None}, "splat_forward: null pointer"),
    ("gsb_splat_forward_rgbd", {"depth_image": None}, "splat_forward_rgbd: null depth_image / alpha_image"),
    ("gsb_splat_forward_rgbd", {"P_cap": -5}, "splat_forward: bad P_cap"),
    ("gsb_splat_forward_rgbd", {"gsid_per_patch": None}, "splat_forward: null pointer"),
    ("gsb_splat_forward_enqueue", {"N": -1}, "splat: bad N/H/W"),
    ("gsb_splat_forward_enqueue", {"bin_ws_bytes": 64}, "splat: bin workspace too small"),
    ("gsb_splat_forward_enqueue", {"P_cap": 0}, "splat_forward: bad P_cap"),
    ("gsb_splat_forward_enqueue", {"us": None}, "splat_forward: null pointer"),
    ("gsb_splat_forward_enqueue", {"final_tau": None}, "splat: null output"),
    ("gsb_splat_forward_enqueue", {"contrib": MIS16}, "splat: misaligned output"),
    ("gsb_splat_forward_enqueue", {"patch_range_per_tile": MIS8}, "splat: misaligned output"),
    ("gsb_splat_forward_enqueue", {"packed_records": MIS16}, "splat: packed_records misaligned"),
    ("gsb_splat_forward_enqueue", {"ws": MIS16}, "splat: ws misaligned"),
    ("gsb_splat_forward_enqueue", {"ws": None}, "splat: workspace too small"),
    ("gsb_splat_forward_enqueue", {"ws_bytes": 64}, "splat: workspace too small"),
    # the surfel frame
    ("gsb_splat_surfel_render", {"H": 0}, "splat: bad N/H/W"),
    ("gsb_splat_surfel_render", {"W": WIDE}, "splat: more than 65535 tiles in a row or column"),
    ("gsb_splat_surfel_render", {"bin_ws": MIS16}, "splat: bin_ws misaligned"),
    ("gsb_splat_surfel_render", {"P": -1}, "splat_surfel: bad P"),
    ("gsb_splat_surfel_render", {"records": None}, "splat_surfel: null pointer"),
    ("gsb_splat_surfel_render", {"image": None}, "splat_surfel: null output"),
    ("gsb_splat_surfel_render", {"normal_image": None}, "splat_surfel: null output"),
    ("gsb_splat_surfel_render", {"alpha_image": MIS16}, "splat_surfel: misaligned output"),
    ("gsb_splat_surfel_render", {"patch_range_per_tile": MIS8}, "splat_surfel: misaligned output"),
    ("gsb_splat_surfel_render", {"records": MIS16}, "splat_surfel: records misaligned"),
    ("gsb_splat_surfel_render", {"ws": MIS16}, "splat_surfel: ws misaligned"),
    ("gsb_splat_surfel_render", {"ws_bytes": 64}, "splat_surfel: workspace too small"),
    ("gsb_splat_surfel_forward", {"N": -1}, "splat: bad N/H/W"),
    ("gsb_splat_surfel_forward", {"H": WIDE}, "splat: more than 65535 tiles in a row or column"),
    ("gsb_splat_surfel_forward", {"bin_ws": MIS16}, "splat: bin_ws misaligned"),
    ("gsb_splat_surfel_forward", {"bin_ws_bytes": 64}, "splat: bin workspace too small"),
    ("gsb_splat_surfel_forward", {"P_cap": 0}, "splat_surfel_forward: bad P_cap"),
    ("gsb_splat_surfel_forward", {"status_host": None}, "splat_surfel_forward: null pointer"),
    ("gsb_splat_surfel_forward", {"records": None}, "splat_surfel_forward: null pointer"),
    ("gsb_splat_surfel_backward", {"P": -1}, "splatB_surfel: bad N/H/W/P"),
    ("gsb_splat_surfel_backward", {"W": WIDE}, "splatB_surfel: more than 65535 tiles in a row or column"),
    ("gsb_splat_surfel_backward", {"rows": None}, "splatB_surfel: null output"),
    ("gsb_splat_surfel_backward", {"ws": MIS16}, "splatB_surfel: workspace too small"),
    ("gsb_splat_surfel_backward", {"ws_bytes": 64}, "splatB_surfel: workspace too small"),
    ("gsb_splat_surfel_backward", {"gsid_per_patch": None}, "splatB_surfel: null pointer"),
    ("gsb_splat_surfel_backward", {"records": MIS16}, "splatB_surfel: misaligned input"),
    ("gsb_splat_surfel_backward", {"patch_range_per_tile": MIS8}, "splatB_surfel: misaligned input"),
    # the colour backward
    ("gsb_splat_backward", {"H": 0}, "splatB: bad N/H/W/P"),
    ("gsb_splat_backward", {"P": -1}, "splatB: bad N/H/W/P"),
    ("gsb_splat_backward", {"moments_out": None, "dloss_dcolors": None}, "splatB: null output"),
    ("gsb_splat_backward", {"ws": None}, "splatB: null pointer"),
    ("gsb_splat_backward", {"ws_bytes": 64}, "splatB: workspace too small"),
    ("gsb_splat_backward", {"dloss_dgammas": None}, "splatB: null pointer"),
    ("gsb_splat_backward", {"packed_records": MIS16}, "splatB: packed_records misaligned"),
    ("gsb_splat_backward_rgbd", {"dloss_ddepths": None}, "splatB_rgbd: null dloss_ddepths"),
    ("gsb_splat_backward_rgbd", {"dloss_dalpha_image": None}, "splatB_rgbd: null pointer"),
    ("gsb_splat_backward_rgbd", {"ws_bytes": 64}, "splatB: workspace too small"),
    ("gsb_splat_backward_abs", {"dloss_dus_abs": None}, "splatB_abs: null dloss_dus_abs"),
    ("gsb_splat_backward_abs", {"N": -1}, "splatB: bad N/H/W/P"),
    ("gsb_splat_backward_rgbd_abs", {"dloss_dus_abs": None}, "splatB_rgbd_abs: null dloss_dus_abs"),
    ("gsb_splat_backward_rgbd_abs", {"dloss_ddepths": None}, "splatB_rgbd: null dloss_ddepths"),
    ("gsb_splat_backward_rgbd_abs", {"depths": None}, "splatB_rgbd: null pointer"),
]


def _param_names():
    """entry point -> its parameter names, from the header's declarations"""
    with open(os.path.join(ROOT, "include", "gsplat_b200.h")) as f:
        src = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    return {m.group(1): [re.findall(r"\w+", p)[-1] for p in m.group(2).split(",")]
            for m in re.finditer(r"\bint\s+(gsb_splat_\w+)\s*\(([^;]*)\)\s*;", src)}


def _run_cases():
    """(rc, gsb_last_error) of every case, in a process without a CUDA device"""
    import ctypes as C
    from easygaussiansplatting_b200 import _lib
    lib = _lib.load()
    names = _param_names()
    status = (C.c_uint32 * 4)()  # written on the host: a real buffer
    base = {"H": 64, "W": 64, "N": 10, "P": 100, "P_cap": 1000, "depth_key_max": 255, "depth_key_cap": 255,
            "ws_bytes": BIG, "bin_ws_bytes": BIG, "status_host": C.addressof(status), "stream": None}
    out = []
    for entry, broken, _ in CASES:
        args = {n: base.get(n, PTR) for n in names[entry]}
        assert set(broken) <= set(args), (entry, broken)
        args.update(broken)
        rc = getattr(lib, entry)(*args.values())
        out.append((rc, lib.gsb_last_error().decode()))
    return out


def test_frame_entry_points_name_the_failed_check():
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
