"""CPU checks of the bilateral-grid colour correction (DESIGN 3.20): the fp64 oracle against the
F.grid_sample composition for the value and both gradients, gradcheck of that composition, the TV
against torch autograd, the identity and clamped-guidance cases, and the C ABI's refusals, profile
ids and register use."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import bilagrid_oracle as bo

PTR = 0x10000000


def _case(M, L, Y, X, B, H, W, seed, lo=-0.2, hi=1.2):
    rng = np.random.default_rng(seed)
    eye = np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], dtype=np.float64).reshape(1, 12, 1, 1, 1)
    grids = eye + 0.3 * rng.standard_normal((M, 12, L, Y, X))
    rgb = rng.uniform(lo, hi, (B, 3, H, W))
    dout = rng.standard_normal((B, 3, H, W))
    return grids, rgb, dout


SIZES = [(16, 16, 8), (3, 5, 1), (4, 3, 1), (1, 4, 3), (7, 1, 5), (1, 1, 1), (2, 2, 2), (5, 7, 3)]


@pytest.mark.parametrize("X,Y,L", SIZES, ids=["X%d-Y%d-L%d" % s for s in SIZES])
def test_oracle_matches_grid_sample(X, Y, L):
    M, B, H, W = 3, 3, 9, 13
    grids, rgb, dout = _case(M, L, Y, X, B, H, W, seed=X * 100 + Y * 10 + L)
    ids = [2, 0, 2]  # a repeated grid: its gradient is the sum of both items'
    ref = bo.slice_grids(grids, rgb, ids, dout)
    tg = torch.tensor(grids, requires_grad=True)
    tr = torch.tensor(rgb, requires_grad=True)
    out = bo.torch_slice(tg, tr, ids)
    out.backward(torch.tensor(dout))
    np.testing.assert_allclose(ref["out"], out.detach().numpy(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(ref["dgrids"], tg.grad.numpy(), rtol=0, atol=1e-11)
    ok = ~ref["ambiguous"][:, None].repeat(3, axis=1)
    np.testing.assert_allclose(ref["drgb"][ok], tr.grad.numpy()[ok], rtol=0, atol=1e-11)
    assert (ref["dgrids_cond"] >= np.abs(ref["dgrids"]) - 1e-12).all()
    assert np.abs(ref["dgrids"][1]).max() == 0.0  # grid 1 is used by no item


def test_grid_sample_composition_passes_gradcheck():
    grids, rgb, _ = _case(2, 3, 2, 3, 2, 4, 5, seed=7, lo=0.05, hi=0.95)
    tg = torch.tensor(grids, requires_grad=True)
    tr = torch.tensor(rgb, requires_grad=True)
    assert torch.autograd.gradcheck(lambda g, r: bo.torch_slice(g, r, [1, 0]), (tg, tr), eps=1e-7, atol=1e-6)


@pytest.mark.parametrize("shape", [(2, 12, 8, 16, 16), (1, 12, 1, 3, 5), (3, 12, 4, 1, 1), (1, 12, 1, 1, 1)])
def test_total_variation_matches_autograd(shape):
    g = np.random.default_rng(sum(shape)).standard_normal(shape)
    tv, grad = bo.total_variation(g)
    t = torch.tensor(g, requires_grad=True)
    ref = 0.0
    for ax in (2, 3, 4):
        if t.shape[ax] > 1:
            ref = ref + (t.diff(dim=ax) ** 2).mean()
    if not isinstance(ref, torch.Tensor):
        assert tv == 0.0 and not grad.any()
        return
    ref.backward()
    assert abs(tv - ref.item()) <= 1e-12 * max(1.0, abs(tv))
    np.testing.assert_allclose(grad, t.grad.numpy(), rtol=0, atol=1e-14)


def test_identity_grid_returns_the_image_and_passes_gradients_through():
    eye = np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], dtype=np.float64).reshape(1, 12, 1, 1, 1)
    grids = np.tile(eye, (2, 1, 8, 16, 16))
    _, rgb, dout = _case(2, 8, 16, 16, 2, 11, 17, seed=3)
    r = bo.slice_grids(grids, rgb, [1, 1], dout)
    np.testing.assert_allclose(r["out"], rgb, rtol=0, atol=1e-15)
    np.testing.assert_allclose(r["drgb"], dout, rtol=0, atol=1e-15)  # a constant grid: dA/dgz = 0


def test_clamped_guidance_has_no_guidance_gradient():
    grids, _, _ = _case(1, 8, 4, 4, 1, 1, 1, seed=5)
    rgb = np.zeros((1, 3, 6, 6))
    rgb[:, :, :3] = -0.5   # g < 0
    rgb[:, :, 3:] = 1.5    # g > 1
    rgb[0, 0, 0, 0] = 3.0  # one channel far out of range, g = 0.897 - 1.402 < 0
    rgb[0, 1:, 0, 0] = -2.0
    dout = np.random.default_rng(1).standard_normal(rgb.shape)
    r = bo.slice_grids(grids, rgb, 0, dout)
    g = np.tensordot(bo.LUMA, rgb[0], axes=1)
    assert ((g < 0) | (g > 1)).all()
    # where g is clamped, A does not move with rgb: dL/drgb is A[:, :3]^T dL/dout, whose columns are
    # the slope of the (then affine) out in each channel
    eps_cols = []
    for k in range(3):
        e = rgb.copy()
        e[0, k] += 1e-3  # stays clamped
        eps_cols.append((bo.slice_grids(grids, e, 0)["out"][0] - r["out"][0]) / 1e-3)
    expect = np.stack([(col * dout[0]).sum(0) for col in eps_cols])
    np.testing.assert_allclose(r["drgb"][0], expect, rtol=1e-9, atol=1e-9)


# ---- the C ABI (no device needed: every refusal returns before a launch)
def _lib():
    from easygaussiansplatting_b200 import _lib as L, build
    build.build()
    return L, L.load()


def _ids(*v):
    return (C.c_int32 * len(v))(*v)


def _slice_args(**kw):
    a = dict(M=4, L=8, Y=16, X=16, grids=PTR, B=2, ids=_ids(0, 3), H=32, W=48, rgb=PTR, out=PTR, stream=None)
    a.update(kw)
    return list(a.values())


SLICE_REFUSALS = [
    ({"M": 0}, "M < 1"), ({"L": 0}, "grid size out of"), ({"X": 65}, "grid size out of"), ({"Y": -1}, "grid size"),
    ({"B": 0}, "batch out of"), ({"B": 65}, "batch out of"), ({"H": 0}, "bad H/W"), ({"W": -2}, "bad H/W"),
    ({"H": 1 << 16, "W": 1 << 15}, "2^31 or more pixels"), ({"ids": None}, "image_ids is null"),
    ({"ids": _ids(0, 4)}, "image id out of"), ({"ids": _ids(-1, 0)}, "image id out of"),
    ({"grids": None}, "null pointer"), ({"rgb": None}, "null pointer"), ({"out": None}, "null pointer"),
    ({"grids": PTR + 2}, "misaligned"), ({"out": PTR + 1}, "misaligned"),
]


@pytest.mark.parametrize("kw,text", SLICE_REFUSALS, ids=[t + "-" + ",".join(k) for k, t in SLICE_REFUSALS])
def test_bilagrid_slice_refusals(kw, text):
    _, lib = _lib()
    assert lib.gsb_bilagrid_slice(*_slice_args(**kw)) == -1
    msg = lib.gsb_last_error().decode()
    assert msg.startswith("argument error: bilagrid_slice: ") and text in msg, msg


def test_bilagrid_backward_and_tv_refusals():
    _, lib = _lib()

    def bwd(**kw):
        a = dict(M=4, L=8, Y=16, X=16, grids=PTR, B=1, ids=_ids(2), H=8, W=8, rgb=PTR, dout=PTR, drgb=PTR,
                 dgrids=PTR, stream=None)
        a.update(kw)
        return lib.gsb_bilagrid_slice_backward(*a.values()), lib.gsb_last_error().decode()

    for kw, text in [({"ids": _ids(4)}, "image id out of"), ({"dgrids": None}, "null pointer"),
                     ({"drgb": None}, "null pointer"), ({"dout": PTR + 2}, "misaligned"), ({"L": 65}, "grid size"),
                     ({"B": 0}, "batch out of")]:
        rc, msg = bwd(**kw)
        assert rc == -1 and "bilagrid_slice_backward: " + text in msg, (kw, msg)
    ws = lib.gsb_bilagrid_tv_workspace_bytes
    assert ws(0, 8, 16, 16) == 0 and ws(1, 65, 16, 16) == 0
    assert 8 <= ws(1, 1, 1, 1) <= ws(300, 8, 16, 16) and ws(300, 8, 16, 16) % 8 == 0
    nb = ws(4, 8, 16, 16)

    def tv(**kw):
        a = dict(M=4, L=8, Y=16, X=16, grids=PTR, tv=PTR, dgrids=None, ws=PTR, ws_bytes=nb, stream=None)
        a.update(kw)
        return lib.gsb_bilagrid_tv(*a.values()), lib.gsb_last_error().decode()

    for kw, text in [({"M": 0}, "M < 1"), ({"X": 0}, "grid size"), ({"tv": None}, "null pointer"),
                     ({"ws": None}, "null pointer"), ({"ws": PTR + 4}, "misaligned"), ({"dgrids": PTR + 2}, "misaligned"),
                     ({"ws_bytes": nb - 1}, "workspace too small")]:
        rc, msg = tv(**kw)
        assert rc == -1 and "bilagrid_tv: " + text in msg, (kw, msg)


def test_bilagrid_profile_ids():
    _, lib = _lib()
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    i = names.index("density_apply_rows")
    assert names[i + 1:i + 5] == ["bilagrid_slice", "bilagrid_slice_backward", "bilagrid_tv", "draw_features"]


def test_bilagrid_kernels_are_sm90a_without_spills():
    L, _ = _lib()
    r = subprocess.run(["cuobjdump", "-res-usage", L.LIB_PATH], capture_output=True, text=True)
    found = dict(re.findall(r"Function (\S*k_bilagrid\w*):\s*\n\s*(REG:.*)", r.stdout))
    names = sorted(re.search(r"(k_bilagrid\w+?)E", k).group(1) for k in found)
    assert names == ["k_bilagrid_slice", "k_bilagrid_slice_bwd", "k_bilagrid_tv", "k_bilagrid_tv_sum"], names
    for name, usage in found.items():
        assert "LOCAL:0 " in usage and "STACK:0 " in usage, (name, usage)
    sass = subprocess.run(["cuobjdump", "-sass", L.LIB_PATH], capture_output=True, text=True).stdout
    assert set(re.findall(r"code for (sm_\w+)", sass)) == {"sm_90a"}


def test_python_surface_checks_without_a_device():
    from easygaussiansplatting_b200 import ops
    from easygaussiansplatting_b200.bilagrid import BilateralGrid
    bil = BilateralGrid(3, grid_X=5, grid_Y=4, grid_L=2, device="cpu")
    assert bil.grids.shape == (3, 12, 2, 4, 5) and bil.num_images == 3
    eye = torch.tensor([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], dtype=torch.float32)
    assert torch.equal(bil.grids.detach().permute(0, 2, 3, 4, 1).reshape(-1, 12), eye.expand(3 * 2 * 4 * 5, 12))
    assert set(bil.state_dict()) == {"grids"}
    with pytest.raises(ValueError, match="CUDA tensor"):
        bil(torch.zeros(3, 4, 4), 0)  # no CPU path
    for bad in ((1, 12, 65, 4, 4), (1, 11, 2, 4, 4), (0, 12, 2, 2, 2), (1, 12, 0, 2, 2)):
        with pytest.raises(ValueError, match="grids must be"):
            ops._bilagrid_dims(bad)
    with pytest.raises(ValueError, match="grids must be"):
        BilateralGrid(2, grid_L=70, device="cpu")
