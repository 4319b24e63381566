"""The host side of a splat frame: splatB's workspace layout from any start, the alignment the
sort and binning workspaces must have, `splatB(records=...)`, and the capacities the two frame
drivers (`ops.splat(capacity=True)` and `GraphedFusedStep`) learn."""
import numpy as np
import pytest
import torch

from easygaussiansplatting_b200.scene import synthetic_scene, upstream_gradient

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def frame(N, W, H, seed, behind=False):
    """one preprocessed frame: (us, cinv2ds, alphas, depths, colors, areas, records), dL/dimage"""
    from easygaussiansplatting_b200 import ops
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=seed)
    if behind:  # every Gaussian behind the camera: no patches
        sc["pws"][:, 2] = -1.0
    al = t(sc["alphas"])
    us, ci, col, d, ar, rec = ops.preprocess(t(sc["pws"]), t(sc["rots"]), t(sc["scales"]), t(sc["shs"]),
                                             t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]), sc["fx"], sc["fy"],
                                             sc["cx"], sc["cy"], W, H, alphas=al)
    return (us, ci, al, d, col, ar, rec), t(upstream_gradient(W, H, seed) * (3.0 * W * H))


def close(a, b):
    """equal up to the order of the backward's float atomics"""
    return torch.allclose(a, b, rtol=1e-4, atol=1e-6 * max(a.abs().max().item(), 1e-30))


@pytest.mark.parametrize("offset", [4, 12, 100])
@pytest.mark.parametrize("empty", [False, True], ids=["P>0", "P=0"])
@pytest.mark.parametrize("given", [False, True], ids=["repack", "records"])
def test_backward_workspace_from_any_start(offset, empty, given):
    """gsb_splat_backward with a ws `offset` bytes past a 256-byte boundary and exactly
    gsb_splat_backward_workspace_bytes long: nothing past its end (or before its start) is written,
    and the gradients are those of an aligned ws"""
    from easygaussiansplatting_b200 import _lib, ops
    lib = _lib.load()
    W, H, N = 200, 120, 3000
    (us, ci, al, d, col, ar, rec), dl = frame(N, W, H, 11, behind=empty)
    out = ops.splat(H, W, us, ci, al, d, col, ar)
    P = out[4].numel()
    assert (P == 0) == empty
    records = rec if given else None
    nbytes = lib.gsb_splat_backward_workspace_bytes(N, H, W, 0 if given else P)
    st = torch.cuda.current_stream().cuda_stream

    def run(buf, off):
        g = [torch.full((N, k), 7.0, device=DEV) for k in (2, 3, 1, 3)]
        _lib.check(lib.gsb_splat_backward(H, W, N, P, us.data_ptr(), ci.data_ptr(), al.data_ptr(), col.data_ptr(),
                                          out[1].data_ptr(), out[2].data_ptr(), out[3].data_ptr(), out[4].data_ptr(),
                                          dl.data_ptr(), None if records is None else records.data_ptr(),
                                          buf.data_ptr() + off, nbytes, *[x.data_ptr() for x in g], None, st), lib)
        return g

    canary = 4096
    buf = torch.full((offset + nbytes + canary,), 0xA5, dtype=torch.uint8, device=DEV)
    assert buf.data_ptr() % 256 == 0
    got = run(buf, offset)
    torch.cuda.synchronize()
    assert bool((buf[:offset] == 0xA5).all()) and bool((buf[offset + nbytes:] == 0xA5).all())
    want = run(torch.empty((nbytes,), dtype=torch.uint8, device=DEV), 0)
    for a, b in zip(want, got):
        if empty:
            assert not a.any() and not b.any()
        else:
            assert close(a, b)


def test_misaligned_workspaces_are_refused_before_any_launch():
    """a ws or bin_ws 4 bytes past a 16-byte boundary is an argument error of every splat entry
    point that takes it, returned before anything is enqueued"""
    from easygaussiansplatting_b200 import _lib, ops
    lib = _lib.load()
    W, H, N = 200, 120, 3000
    (us, ci, al, d, col, ar, rec), _ = frame(N, W, H, 12)
    out = ops.splat(H, W, us, ci, al, d.clone(), col, ar.clone())
    P = out[4].numel()
    torch.cuda.synchronize()
    st = torch.cuda.current_stream().cuda_stream
    bin_bytes = lib.gsb_splat_bin_workspace_bytes(N)
    ws_bytes = lib.gsb_splat_workspace_bytes(N, H, W, P + 1)  # (the forward's P_cap)
    bin_buf = torch.full((bin_bytes + 16,), 0xA5, dtype=torch.uint8, device=DEV)
    ws_buf = torch.full((ws_bytes + 16,), 0xA5, dtype=torch.uint8, device=DEV)
    outs = [torch.empty_like(x) for x in out[:4]] + [torch.empty((P + 1,), dtype=torch.int32, device=DEV)]
    status = torch.zeros(4, dtype=torch.int32).pin_memory()
    p = lambda x: x.data_ptr()
    dd, aa = d.clone(), ar.clone()

    def bin_(bo):
        return lib.gsb_splat_bin(H, W, N, p(us), p(dd), p(aa), p(bin_buf) + bo, bin_bytes, None, None, st)

    def render(bo, wo):
        return lib.gsb_splat_render(H, W, N, P, 0xFFFFFFFF, p(us), p(ci), p(al), p(dd), p(col), None,
                                    p(bin_buf) + bo, p(ws_buf) + wo, ws_bytes, *map(p, outs), st)

    def forward(fn, bo, wo):
        return fn(H, W, N, p(us), p(ci), p(al), p(dd), p(col), p(aa), p(rec), P + 1, 0xFFFFFFFF,
                  p(bin_buf) + bo, bin_bytes, p(ws_buf) + wo, ws_bytes, *map(p, outs), status.data_ptr(), st)

    calls = [lambda: bin_(4), lambda: render(4, 0), lambda: render(0, 4)]
    for fn in (lib.gsb_splat_forward, lib.gsb_splat_forward_enqueue):
        calls += [lambda fn=fn: forward(fn, 4, 0), lambda fn=fn: forward(fn, 0, 4)]
    # (gsb_splat_bin's P_host is NULL above: the alignment error comes first)
    before = lib.gsb_profile_launches(-1)
    for call in calls:
        assert call() == -1
        assert b"misaligned" in lib.gsb_last_error()
    torch.cuda.synchronize()
    assert lib.gsb_profile_launches(-1) == before
    assert torch.equal(dd, d) and torch.equal(aa, ar)  # nothing was binned
    assert bool((ws_buf == 0xA5).all()) and bool((bin_buf == 0xA5).all())


def test_splatB_takes_the_forward_records():
    """splatB(records=rec) equals splatB reading the same records from what `splat` attached to
    gsid_per_patch, in both output modes, and packs nothing even when that handle is gone"""
    from easygaussiansplatting_b200 import _lib, ops
    lib = _lib.load()
    pack = [lib.gsb_profile_kernel_name(i) for i in range(lib.gsb_profile_kernels())].index(b"pack_records")
    W, H, N = 320, 240, 20000
    (us, ci, al, d, col, ar, rec), dl = frame(N, W, H, 13)
    out = ops.splat(H, W, us, ci, al, d, col, ar, records=rec)
    assert ops._cached_records(out[4], (us, ci, al, col)) == rec.data_ptr()
    args = (H, W, us, ci, al, d, col, out[1], out[2], out[3], out[4], dl)
    for moments_only in (False, True):
        cached = ops.splatB(*args, moments_only=moments_only)
        given = ops.splatB(*args, moments_only=moments_only, records=rec)
        for a, b in zip(*[x if isinstance(x, list) else [x] for x in (cached, given)]):
            assert close(a, b)
    ops.forget_records(out[4])
    before = lib.gsb_profile_launches(pack)
    m = ops.splatB(*args, moments_only=True, records=rec)
    assert lib.gsb_profile_launches(pack) == before
    assert close(m, ops.splatB(*args, moments_only=True))  # (re-packed)
    assert lib.gsb_profile_launches(pack) == before + 1
    with pytest.raises(ValueError, match="records"):
        ops.splatB(*args, records=rec[:-1])


# what both drivers learnt on this scene while each had its own copy of the frame (H100 80GB HBM3)
GRAPHED_CAPS = [79181, 16383]
SPLAT_CAPS_EXACT = [66667, 16383]
SPLAT_CAPS_CAPACITY = [66667, 16383]


def test_learnt_capacities_are_unchanged():
    """GraphedFusedStep (1.5x head-room, depth bound from the depths) and ops.splat(capacity=True)
    (1.25x, depth bound from the binning) learn the same bounds as before on one fixed scene"""
    from easygaussiansplatting_b200 import ops
    from easygaussiansplatting_b200.gsfunction import Camera
    from easygaussiansplatting_b200.graphed import GraphedFusedStep
    W, H, N = 320, 240, 20000
    sc = synthetic_scene(N, W, H, sh_dim=12, seed=6)
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]))
    P = {k: t(sc[k]) for k in ("pws", "shs", "scales", "rots")}
    al = t(sc["alphas"][:, None])
    step = GraphedFusedStep(P["pws"], P["shs"], al, P["scales"], P["rots"], cam)
    assert [step.P_cap, step.dk_cap] == GRAPHED_CAPS
    us, ci, col, dep, ar = ops.preprocess(P["pws"], P["rots"], P["scales"], P["shs"], cam.Rcw, cam.tcw, cam.twc,
                                          cam.fx, cam.fy, cam.cx, cam.cy, W, H)
    ops._CAPACITY.clear()
    key = (0, H, W, N)
    try:
        ops.splat(H, W, us, ci, al, dep, col, ar, capacity=True)
        assert list(ops._CAPACITY[key]) == SPLAT_CAPS_EXACT
        ops.splat(H, W, us, ci, al, dep, col, ar, capacity=True)
        assert list(ops._CAPACITY[key]) == SPLAT_CAPS_CAPACITY
    finally:
        ops._CAPACITY.clear()
