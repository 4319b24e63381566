"""The fused per-Gaussian chain training runs -- preprocess(alphas=...) -> splat(records=...,
capacity=True) -> splatB(moments_only=True) -> preprocessB(moments=...), plus sh_grad_expand --
against the fp64 oracle at every SH degree, at N that leave the last 128-Gaussian CTA full,
almost empty or almost full, and at odd N whose gradient bucket views start off the 16-byte grid.

Also the alignment contract of the op layer: any contiguous float32 / int32 tensor is accepted,
including a view one element into its storage (what packing per-Gaussian state into one flat
buffer produces).  Such a view takes the kernels' scalar paths and must give bit-identical
results to the aligned call.

Tolerances (fp32 device arithmetic vs the fp64 oracle on identical fp32 inputs) follow
test_fused_math_cpu.py, which checks the same per-Gaussian math on the host."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from easygaussiansplatting_b200.scene import ring_camera, upstream_gradient
from test_gpu_fused import n, scene, t
from test_gpu_parity import check_splat_vs_oracle

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
W, H = 320, 240
K3S = (1, 4, 9, 16)
NS = (1, 127, 129, 20001)   # N mod 128 = 1, 127, 1, 33; 20001 is odd: off-grid bucket views
Z_BAND = 1e-5               # |z - 0.2| below this: the cull may go either way in fp32


def f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def edge_scene(N, k3, seed=1):
    """scene() with an odd seed (rotated camera, un-normalised quaternions); for N >= 64 its
    last rows are edge cases: quaternion 0, scale 0, depths a few ulp either side of 0.2, an
    infinite scale (NaN 2D determinant) and centres outside the 1.3 tan_fov cone."""
    sc = scene(N, W, H, 3 * k3, seed)
    if N == 1:  # (scene() sends its one row behind the camera)
        sc["pws"][0] = f32(sc["Rcw"].astype(np.float64).T @ (np.array([0.05, -0.02, 2.5]) - sc["tcw"]))
    if N < 64:
        return sc
    R, tc = sc["Rcw"].astype(np.float64), sc["tcw"].astype(np.float64)
    tfx, tfy = W / (2 * sc["fx"]), H / (2 * sc["fy"])
    z02 = np.float32(0.2)
    pcs = [(0.1, 0.05, 2.0), (-0.2, 0.1, 3.0)]
    pcs += [(0.01, 0.02, float(z)) for z in (np.nextafter(np.nextafter(z02, 0), 0), np.nextafter(z02, 0), z02,
                                             np.nextafter(z02, 1), np.nextafter(np.nextafter(z02, 1), 1))]
    pcs += [(0.0, 0.0, 2.0), (3.0 * 2.0 * tfx, 0.1, 2.0), (0.1, -3.0 * 4.0 * tfy, 4.0)]
    E = len(pcs)
    rows = np.arange(N - E, N)
    sc["pws"][rows] = f32([R.T @ (np.array(p) - tc) for p in pcs])
    sc["rots"][rows] = f32([1.0, 0.1, -0.2, 0.05])
    sc["scales"][rows] = 0.05
    sc["rots"][rows[0]] = 0.0                        # quaternion 0
    sc["scales"][rows[1]] = 0.0                      # scale 0
    sc["scales"][rows[7]] = [np.inf, 0.05, 0.05]     # cov2d inf -> 1/det NaN -> culled
    sc["edge_rows"] = rows
    sc["nan_det_row"] = rows[7]
    return sc


def params(sc):
    return [t(sc[k]) for k in ("pws", "rots", "scales", "shs", "Rcw", "tcw", "twc")]


def cam_args(sc):
    return (sc["fx"], sc["fy"], sc["cx"], sc["cy"], W, H)


def oracle_stages(sc, Wi=W, Hi=H):
    us, pcs, depths, Ju = orc.project(sc["pws"], sc["Rcw"], sc["tcw"], sc["fx"], sc["fy"], sc["cx"], sc["cy"])
    d32 = f32(depths)
    c3, J3r, J3s = orc.compute_cov3d(sc["rots"], sc["scales"], d32)
    c2, J2c, J2p = orc.compute_cov2d(f32(c3), f32(pcs), sc["Rcw"], d32, sc["fx"], sc["fy"], Wi, Hi)
    col, Jcs, Jcp = orc.sh2color(sc["shs"], sc["pws"], sc["twc"])
    ci, areas, Jci = orc.inverse_cov2d(f32(c2), d32)   # d32: NaN determinant -> -1
    z64 = sc["pws"].astype(np.float64) @ sc["Rcw"].astype(np.float64)[2] + float(sc["tcw"][2])
    return dict(us=us, depths=d32, depth64=depths, ci=ci, col=col, areas=areas, band=np.abs(z64 - 0.2) < Z_BAND,
                J=(Ju, J3r, J3s, J2c, J2p, Jcs, Jcp, Jci))


def close(got, ref, name, rtol=3e-5, atol_scale=6e-6, rows=None):
    """elementwise |got - ref| <= rtol |ref| + atol_scale max|ref| (over `rows`)"""
    got = np.asarray(got, np.float64).reshape(ref.shape)
    if rows is not None:
        got, ref = got[rows], ref[rows]
    if not ref.size:
        return
    scale = max(np.abs(ref).max(), 1e-30)
    excess = np.abs(got - ref) - (rtol * np.abs(ref) + atol_scale * scale)
    i = np.argmax(excess)
    assert excess.flat[i] <= 0, "%s: got %r want %r (scale %g)" % (name, got.flat[i], ref.flat[i], scale)


def norm_err(got, ref, rows=None):
    got = np.asarray(got, np.float64).reshape(ref.shape)
    if rows is not None:
        got, ref = got[rows], ref[rows]
    if not ref.size:
        return 0.0
    return np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30)


def finite_rows(ref):
    """rows where the oracle chain is finite (0 * inf Jacobian entries of the infinite-scale row,
    which the fused kernel never forms: it skips culled rows)"""
    return np.all([np.isfinite(ref[k]).all(axis=1) for k in ("pws", "shs", "scales", "rots")], axis=0)


def shifted(x):
    """x as a contiguous view one element into a fresh buffer (same values; 4 bytes past a
    16-byte boundary, so every vector access on it is misaligned)"""
    buf = torch.empty(x.numel() + 1, dtype=x.dtype, device=x.device)
    v = buf[1:].view(x.shape)
    v.copy_(x)
    assert v.is_contiguous() and v.data_ptr() % 16 == 4
    return v


def _junk(dtype):
    return float("nan") if dtype.is_floating_point else -7


def shifted_empty(shape, dtype=torch.float32):
    """an output one element past a 16-byte boundary, filled with junk"""
    v = torch.full((int(np.prod(shape)) + 1,), _junk(dtype), dtype=dtype, device=DEV)[1:].view(shape)
    assert v.data_ptr() % 16 == 4
    return v


def aligned_empty(shape, dtype=torch.float32):
    v = torch.full(shape, _junk(dtype), dtype=dtype, device=DEV)
    assert v.data_ptr() % 16 == 0
    return v


# ---------------------------------------------------------------- 1. fused forward
@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("k3", K3S)
def test_preprocess_vs_oracle(k3, N):
    from easygaussiansplatting_b200 import ops
    sc = edge_scene(N, k3)
    us, ci, col, d, ar = [n(x) for x in ops.preprocess(*params(sc), *cam_args(sc))]
    o = oracle_stages(sc)
    band = o["band"]
    keep_g, keep_o = d > 0, o["depths"] > 0
    assert np.array_equal(keep_g[~band], keep_o[~band])
    if "nan_det_row" in sc:
        r = sc["nan_det_row"]
        assert not band[r] and not keep_o[r] and not keep_g[r] and d[r] == -1.0
        assert band[sc["edge_rows"][2:7]].all()   # the rows a few ulp either side of z = 0.2
    both = keep_g & keep_o
    close(us, o["us"], "us", rows=both)
    close(d, o["depth64"], "depths", rows=both)
    close(col, o["col"], "colors")                       # colours are not gated by the cull
    close(ci, o["ci"], "cinv2ds", rtol=1e-4, atol_scale=2e-5, rows=both)
    # radius from the fused fp32 cov2d vs the oracle's fp64 one: equal except where 3 sqrt() sits
    # within fp32 rounding of an integer (under 0.2 % of the rows; one row at the small N)
    diff = ar[both] != o["areas"][both]
    assert diff.sum() <= max(1, 2e-3 * diff.size) and np.abs(ar[both] - o["areas"][both]).max(initial=0) <= 1
    # culled rows are exactly 0 in us, cinv2ds and areas; their depth is -1
    assert not us[~keep_g].any() and not ci[~keep_g].any() and not ar[~keep_g].any()
    assert np.all(d[~keep_g] == -1.0)


# ---------------------------------------------------------------- 2. alignment twins
PARAM_NAMES = ("pws", "rots", "scales", "shs")


@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("k3", K3S)
def test_preprocess_offset_views_bit_identical(k3, N):
    """pws / rots / scales / shs (and the upstream gradients) as views one float into their
    storage: the scalar load paths give the same bits as the vector ones.  On the output side,
    gsb_preprocess_backward writing into outputs one float past a 16-byte boundary (the scalar
    drots store and the scalar dsh tile flush) gives the same bits as writing into aligned ones,
    and both equal ops.preprocessB (whose bucket views are off-grid for odd N and k3 in {1, 9})."""
    from easygaussiansplatting_b200 import _lib, ops
    sc = edge_scene(N, k3, seed=3)
    P = params(sc)
    cam = cam_args(sc)
    rng = np.random.default_rng(N + k3)
    gu, gci, gcol = (t(rng.normal(size=(N, k)).astype(np.float32)) for k in (2, 3, 3))
    fwd = ops.preprocess(*P, *cam)
    bwd = ops.preprocessB(*P, *cam, gu, gci, gcol)
    mom = t(rng.normal(size=(N, 9)).astype(np.float32))
    bwdm = ops.preprocessB(*P, *cam, None, None, None, moments=mom, cinv2ds=fwd[1])
    for which in [(i,) for i in range(4)] + [(0, 1, 2, 3)]:
        Q = [shifted(p) if i in which else p for i, p in enumerate(P[:4])] + P[4:]
        for a, b in zip(fwd, ops.preprocess(*Q, *cam)):
            assert torch.equal(a, b), ("forward", [PARAM_NAMES[i] for i in which])
        for a, b in zip(bwd, ops.preprocessB(*Q, *cam, shifted(gu), shifted(gci), shifted(gcol))):
            assert torch.equal(a, b), ("backward", [PARAM_NAMES[i] for i in which])
        for a, b in zip(bwdm, ops.preprocessB(*Q, *cam, None, None, None, moments=shifted(mom),
                                              cinv2ds=shifted(fwd[1]))):
            assert torch.equal(a, b), ("moment backward", [PARAM_NAMES[i] for i in which])
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    shapes = dict(pws=(N, 3), shs=(N, 3 * k3), scales=(N, 3), rots=(N, 4), dus=(N, 2), dal=(N,))
    for moments in (False, True):
        want = bwdm if moments else bwd
        got = []
        for alloc in (aligned_empty, shifted_empty):
            o = {k: alloc(s) for k, s in shapes.items()}
            up = (None, None, None, mom.data_ptr(), fwd[1].data_ptr(), o["dus"].data_ptr(), o["dal"].data_ptr()) \
                if moments else (gu.data_ptr(), gci.data_ptr(), gcol.data_ptr(), None, None, None, None)
            _lib.check(lib.gsb_preprocess_backward(
                N, k3, *[p.data_ptr() for p in P], *[float(c) for c in cam], *up[:3], o["pws"].data_ptr(),
                o["shs"].data_ptr(), o["scales"].data_ptr(), o["rots"].data_ptr(), *up[3:], st), lib)
            got.append(o)
        for k in ("pws", "shs", "scales", "rots") + (("dus", "dal") if moments else ()):
            assert torch.equal(got[0][k], got[1][k]), ("output offset", moments, k)
        for k, w in zip(("pws", "shs", "scales", "rots", "dus", "dal"), want):
            assert torch.equal(got[1][k], w), ("vs ops.preprocessB", moments, k)


# ---------------------------------------------------------------- 3. plain backward
@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("k3", K3S)
def test_preprocess_backward_vs_oracle(k3, N):
    from easygaussiansplatting_b200 import ops
    sc = edge_scene(N, k3, seed=5)
    o = oracle_stages(sc)
    d = n(ops.preprocess(*params(sc), *cam_args(sc))[3])
    keep = (o["depths"] > 0) & (d > 0)
    rng = np.random.default_rng(7 * N + k3)
    gu = rng.normal(size=(N, 1, 2)).astype(np.float32)
    gci = rng.normal(size=(N, 1, 3)).astype(np.float32) * 10
    gcol = rng.normal(size=(N, 1, 3)).astype(np.float32)
    gal = np.zeros((N, 1, 1), np.float32)
    col_only = rng.random(N) < 0.01              # the `any` early exit: colour gradient only
    if N > 1:
        col_only[rng.integers(N)] = True
    gu[col_only] = 0; gci[col_only] = 0
    gu[~keep] = 0; gci[~keep] = 0; gcol[~keep] = 0   # culled Gaussians have no patches
    ref = orc.chain_backward(sc["Rcw"], gu, gci, gal, gcol, *o["J"])
    gpw, gsh, gs, gq = [n(x) for x in ops.preprocessB(*params(sc), *cam_args(sc), t(gu), t(gci), t(gcol))]
    fin = finite_rows(ref)
    assert fin[keep].all()
    for got, name in ((gpw, "pws"), (gsh, "shs"), (gs, "scales"), (gq, "rots")):
        e = norm_err(got, ref[name], rows=fin)
        assert e <= 2e-5, (name, e)
    close(gsh, ref["shs"], "dshs", rtol=1e-5, atol_scale=1e-6, rows=fin)
    # rows without upstream geometry gradient: scales / rots exactly 0, pws the colour term alone
    co = col_only & keep
    assert not gs[co].any() and not gq[co].any() and not gs[~keep].any() and not gq[~keep].any()
    assert not gpw[~keep].any() and not gsh[~keep].any()
    close(gpw, ref["pws"], "dpws (colour only)", rtol=1e-5, atol_scale=1e-6, rows=co)


# ---------------------------------------------------------------- 4. moment rows
def moment_case(sc, N, k3, seed):
    """forward cinv2ds + random moment rows; ~5 % of the kept rows untouched (m0 = m1 = 0), some
    of those with an inf / NaN conic.  Culled rows get no moments (no patches)."""
    from easygaussiansplatting_b200 import ops
    fwd = ops.preprocess(*params(sc), *cam_args(sc))
    ci = n(fwd[1]).copy()
    keep = n(fwd[3]) > 0
    rng = np.random.default_rng(seed)
    m = rng.normal(size=(N, 9)).astype(np.float32)
    m[:, 2:5] *= 10
    m[~keep] = 0
    none = keep & (rng.random(N) < 0.05)
    m[none, 0:2] = 0
    bad = np.flatnonzero(none)[::3]
    ci[bad[0::2]] = np.inf
    ci[bad[1::2], 1] = np.nan
    return m, ci, keep, none


@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("k3", K3S)
def test_preprocess_backward_moments_vs_oracle(k3, N):
    from easygaussiansplatting_b200 import ops
    sc = edge_scene(N, k3, seed=7)
    o = oracle_stages(sc)
    m, ci, keep, none = moment_case(sc, N, k3, 11 * N + k3)
    gpw, gsh, gs, gq, dus, dal = [n(x) for x in ops.preprocessB(*params(sc), *cam_args(sc), None, None, None,
                                                              moments=t(m), cinv2ds=t(ci))]
    # expected upstream gradients in fp64 from the fp32 inputs (k_preprocess_bwd's conversion)
    md, cd = m.astype(np.float64), ci.astype(np.float64)
    with np.errstate(invalid="ignore"):
        A, B, Cc = cd[:, 0], cd[:, 1], cd[:, 2]
        gu = -np.stack([A * md[:, 0] + B * md[:, 1], B * md[:, 0] + Cc * md[:, 1]], axis=1)
        bound = 2.0 ** -22 * np.stack([np.abs(A * md[:, 0]) + np.abs(B * md[:, 1]),
                                       np.abs(B * md[:, 0]) + np.abs(Cc * md[:, 1])], axis=1)
    gu[none] = 0
    bound[none] = 0
    assert np.all(dus[none] == 0) and not np.isnan(dus).any()
    assert np.all(np.abs(dus[~none] - gu[~none]) <= bound[~none]), "dus"
    assert np.array_equal(dal, m[:, 5])                                   # pass-through, bit-exact
    gci = np.stack([-0.5 * md[:, 2], -md[:, 3], -0.5 * md[:, 4]], axis=1)
    ref = orc.chain_backward(sc["Rcw"], gu[:, None], gci[:, None], md[:, 5:6, None], md[:, None, 6:9], *o["J"])
    rows = keep & (o["depths"] > 0) & finite_rows(ref)
    for got, name in ((gpw, "pws"), (gsh, "shs"), (gs, "scales"), (gq, "rots")):
        e = norm_err(got, ref[name], rows=rows)
        assert e <= 2e-5, (name, e)


@pytest.mark.parametrize("N", [128, 129, 20000, 20001])
@pytest.mark.parametrize("k3", K3S)
def test_compact_bucket_equals_full(k3, N):
    """compact=True: the flat bucket [dpws | dscales | drots | dalphas] holds the same bits as the
    separate outputs, and there is no dshs.  drots starts 6N floats in: 16-byte aligned for even N
    (vector store), 8 bytes off for odd N (scalar store)."""
    from easygaussiansplatting_b200 import ops
    sc = edge_scene(N, k3, seed=7)
    m, ci, _, _ = moment_case(sc, N, k3, 17 * N + k3)
    full = ops.preprocessB(*params(sc), *cam_args(sc), None, None, None, moments=t(m), cinv2ds=t(ci))
    comp = ops.preprocessB(*params(sc), *cam_args(sc), None, None, None, moments=t(m), cinv2ds=t(ci), compact=True)
    assert comp[1] is None
    assert (comp[3].data_ptr() % 16 == 0) == (N % 2 == 0)
    for i in (0, 2, 3, 4, 5):
        assert torch.equal(full[i], comp[i]), i


# ---------------------------------------------------------------- 5. sh_grad_expand
@pytest.mark.parametrize("V", [1, 3, 8])
@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("k3", K3S)
def test_sh_grad_expand_vs_fp64(k3, N, V):
    from easygaussiansplatting_b200 import ops
    sc = edge_scene(N, k3, seed=9)
    rng = np.random.default_rng(13 * N + V)
    twcs = f32([ring_camera(v, 8)[2] for v in range(V)])
    g = rng.normal(size=(V, N, 3)).astype(np.float32)
    ref = np.zeros((N, k3, 3))
    for v in range(V):
        Js = orc.sh2color(sc["shs"], sc["pws"], twcs[v])[1]            # [N,1,k]
        ref += Js[:, 0, :, None] * g[v][:, None, :].astype(np.float64)
    ref = ref.reshape(N, 3 * k3)
    got = n(ops.sh_grad_expand(t(sc["pws"]), t(twcs), t(g), k3))
    assert norm_err(got, ref) <= 1e-5, norm_err(got, ref)
    close(got, ref, "dshs", rtol=1e-4, atol_scale=1e-5)
    if V == 1:  # the same basis as the per-Gaussian backward's dL/dsh row, up to FMA contraction
        P = params(sc)
        ci = ops.preprocess(*P, *cam_args(sc))[1]
        m = np.zeros((N, 9), np.float32)
        m[:, 6:9] = g[0]
        Q = P[:6] + [t(twcs[0])]
        dshs = n(ops.preprocessB(*Q, *cam_args(sc), None, None, None, moments=t(m), cinv2ds=ci)[1])
        assert norm_err(got, dshs.astype(np.float64)) <= 1e-6


def test_sh_grad_expand_validates_out():
    from easygaussiansplatting_b200 import ops
    N, k3, V = 300, 9, 2
    rng = np.random.default_rng(0)
    pws = t(rng.normal(size=(N, 3)).astype(np.float32) + [0, 0, 3])
    twcs = t(rng.normal(size=(V, 3)).astype(np.float32))
    g = t(rng.normal(size=(V, N, 3)).astype(np.float32))
    want = ops.sh_grad_expand(pws, twcs, g, k3)
    out = torch.full((N, 3 * k3), np.nan, device=DEV)
    assert ops.sh_grad_expand(pws, twcs, g, k3, out=out) is out and torch.equal(out, want)
    for bad, err in ((torch.empty((N - 1, 3 * k3), device=DEV), ValueError),
                     (torch.empty((N, 3 * k3 + 1), device=DEV), ValueError),
                     (torch.empty((N * 3 * k3,), device=DEV), ValueError),
                     (torch.empty((3 * k3, N), device=DEV).t(), ValueError),
                     (torch.empty((N, 3 * k3), dtype=torch.float64, device=DEV), TypeError),
                     (torch.empty((N, 3 * k3)), ValueError)):
        with pytest.raises(err):
            ops.sh_grad_expand(pws, twcs, g, k3, out=bad)


# ---------------------------------------------------------------- 6. end to end
@pytest.mark.parametrize("k3,N,Wi,Hi", [(1, 3000, 250, 130), (4, 4000, 979, 546), (9, 2000, 320, 240),
                                        (16, 20000, 320, 240)])
def test_fused_function_end_to_end_vs_oracle(k3, N, Wi, Hi):
    """GSFunctionFused (the records + capacity forward, the moment-row backward) against the
    oracle: the image through check_splat_vs_oracle on the fused forward's own outputs, and the
    parameter gradients through the oracle's rasterizer backward and fp64 Jacobian chain."""
    from easygaussiansplatting_b200 import ops
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused
    sc = scene(N, Wi, Hi, 3 * k3, N + 1)
    Pw = [t(sc[k]) for k in ("pws", "rots", "scales", "shs", "Rcw", "tcw", "twc")]
    camargs = (sc["fx"], sc["fy"], sc["cx"], sc["cy"], Wi, Hi)
    al = t(sc["alphas"])
    us, ci, col, d, ar = ops.preprocess(*Pw, *camargs)
    # (also checks splatB against the oracle's rasterizer backward on these inputs; culls d / ar in place)
    fwd_out, ref = check_splat_vs_oracle(Hi, Wi, us, ci, al, d, col, ar, seed=k3)
    d_binned = n(d)
    ops._CAPACITY.clear()
    cam = Camera(Wi, Hi, sc["fx"], sc["fy"], sc["cx"], sc["cy"], Pw[4], Pw[5], Pw[6])
    dl = upstream_gradient(Wi, Hi, k3) * (3.0 * Wi * Hi)
    got = {}
    for rep in range(2):   # the first frame learns the capacities, the second runs the capacity path
        leaves = {k: t(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
        alr = t(sc["alphas"][:, None]).requires_grad_()
        us0 = torch.zeros((N, 2), device=DEV, requires_grad=True)
        image, mask = GSFunctionFused.apply(leaves["pws"], leaves["shs"], alr, leaves["scales"], leaves["rots"],
                                            us0, cam)
        image.backward(t(dl))
        got = dict(image=image.detach(), mask=n(mask), dpws=n(leaves["pws"].grad), dshs=n(leaves["shs"].grad),
                   dscales=n(leaves["scales"].grad), drots=n(leaves["rots"].grad), dalphas=n(alr.grad)[:, 0],
                   dus=n(us0.grad))
        assert torch.equal(got["image"], fwd_out[0])
    # mask: the oracle's depth > 0.2 after its culls (projection and NaN determinant in fp64, then
    # the binning's "touches no tile", which check_splat_vs_oracle matched bit for bit)
    o = oracle_stages(sc, Wi, Hi)
    band = o["band"]
    want_mask = (o["depths"] > 0.2) & (d_binned > 0.2)
    assert np.array_equal(got["mask"][~band], want_mask[~band])
    # gradients: oracle rasterizer backward -> fp64 chain with Jacobians from the fp32 parameters
    du, dc, da, dcol, amb = orc.splat_backward(Hi, Wi, n(us), n(ci), n(al), n(col), ref, dl, return_ambiguous=True)
    chain = orc.chain_backward(sc["Rcw"], du, dc, da, dcol, *o["J"])
    strict = ~(amb | band)
    for name, key in (("dpws", "pws"), ("dshs", "shs"), ("dscales", "scales"), ("drots", "rots"),
                      ("dalphas", "alphas"), ("dus", "us")):
        want = chain[key].reshape(N, -1)
        g = got[name].reshape(N, -1).astype(np.float64)
        s = max(np.abs(want).max(), 1e-30)
        err = np.abs(g - want).max(axis=1) / s
        assert err[strict].max(initial=0) <= 1e-4, (name, err[strict].max(initial=0))
        assert err[~band].max(initial=0) <= 5e-3, (name, err[~band].max(initial=0))


# ---------------------------------------------------------------- 8. misaligned views at the op surface
@pytest.mark.parametrize("N,Wi,Hi", [(3001, 320, 240), (20001, 979, 546)])
def test_splat_splatB_density_accept_offset_views(N, Wi, Hi):
    """splat with us / areas / depths, splatB with patch_range_per_tile, preprocessB with
    dloss_dus and density.accumulate with dloss_dus, each given as a contiguous view one
    element into its storage: bit-identical to the aligned call (splat's in-place culls
    included, written through the view), except splatB's moment rows, which are sums of float
    atomics and agree to rounding."""
    from easygaussiansplatting_b200 import density, ops
    sc = scene(N, Wi, Hi, 12, 3)
    P = [t(sc[k]) for k in ("pws", "rots", "scales", "shs", "Rcw", "tcw", "twc")]
    camargs = (sc["fx"], sc["fy"], sc["cx"], sc["cy"], Wi, Hi)
    al = t(sc["alphas"])
    us, ci, col, d, ar = ops.preprocess(*P, *camargs)
    d0, ar0 = d.clone(), ar.clone()
    a = ops.splat(Hi, Wi, us, ci, al, d0, col, ar0)
    assert (d0 < 0).sum() > (d < 0).sum()   # the binning culled Gaussians that touch no tile
    for which in ("us", "areas", "depths", "all"):
        u1 = shifted(us) if which in ("us", "all") else us
        d1 = shifted(d) if which in ("depths", "all") else d.clone()
        ar1 = shifted(ar) if which in ("areas", "all") else ar.clone()
        b = ops.splat(Hi, Wi, u1, ci, al, d1, col, ar1)
        for x, y in zip(a, b):
            assert torch.equal(x, y), which
        assert torch.equal(d1, d0) and torch.equal(ar1, ar0), which
    dl = t(upstream_gradient(Wi, Hi, 2) * (3.0 * Wi * Hi))
    image, contrib, ftau, ranges, gsid = a
    ops.forget_records(gsid)
    g0 = ops.splatB(Hi, Wi, us, ci, al, d0, col, contrib, ftau, ranges, gsid, dl, moments_only=True)
    g1 = ops.splatB(Hi, Wi, shifted(us), ci, al, d0, col, contrib, ftau, shifted(ranges), gsid, dl,
                    moments_only=True)
    # (the moment rows are sums of float atomics whose order varies from run to run, so two
    # calls agree to rounding, not bitwise; the same rows must be touched)
    assert torch.equal(g0 != 0, g1 != 0)
    assert float((g0 - g1).abs().max() / g0.abs().max()) <= 1e-5
    gu = t(np.random.default_rng(1).normal(size=(N, 2)).astype(np.float32))
    gc, gcol = torch.ones((N, 3), device=DEV), torch.ones((N, 3), device=DEV)
    x = ops.preprocessB(*P, *camargs, gu, gc, gcol)
    y = ops.preprocessB(*P, *camargs, shifted(gu), gc, gcol)
    for p, q in zip(x, y):
        assert torch.equal(p, q)
    mask = d0 > 0
    acc0, acc1 = torch.empty((N, 1), device=DEV), torch.empty((N, 1), device=DEV)
    cnt0, cnt1 = torch.empty(N, dtype=torch.int32, device=DEV), torch.empty(N, dtype=torch.int32, device=DEV)
    for first in (1, 0, 0):
        density.accumulate(gu, mask, acc0, cnt0, first)
        density.accumulate(shifted(gu), mask, acc1, cnt1, first)
    assert torch.equal(acc0, acc1) and torch.equal(cnt0, cnt1)
    assert torch.equal(cnt0, 3 * mask.to(torch.int32))


def test_splat_rejects_misaligned_outputs_at_the_abi():
    """the C ABI's fresh outputs of the rasterizer (image planes 16 B, tile ranges 8 B) are
    checked, not silently mis-stored"""
    from easygaussiansplatting_b200 import _lib, ops
    N, Wi, Hi = 500, 64, 48
    sc = scene(N, Wi, Hi, 3, 1)
    us, ci, col, d, ar = ops.preprocess(*[t(sc[k]) for k in ("pws", "rots", "scales", "shs", "Rcw", "tcw", "twc")],
                                        sc["fx"], sc["fy"], sc["cx"], sc["cy"], Wi, Hi)
    al = t(sc["alphas"])
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    bin_bytes = lib.gsb_splat_bin_workspace_bytes(N)
    bin_ws = torch.empty(bin_bytes, dtype=torch.uint8, device=DEV)
    P, dk = C.c_int64(0), C.c_uint32(0)
    _lib.check(lib.gsb_splat_bin(Hi, Wi, N, us.data_ptr(), d.data_ptr(), ar.data_ptr(), bin_ws.data_ptr(), bin_bytes,
                                 C.byref(P), C.byref(dk), st), lib)
    P = int(P.value)
    ws_bytes = lib.gsb_splat_workspace_bytes(N, Hi, Wi, P)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
    T = ((Wi + 15) // 16) * ((Hi + 15) // 16)
    gsid = torch.empty(max(P, 1), dtype=torch.int32, device=DEV)

    def render(img, con, ft, rg):
        return lib.gsb_splat_render(Hi, Wi, N, P, dk.value, us.data_ptr(), ci.data_ptr(), al.data_ptr(), d.data_ptr(),
                                    col.data_ptr(), None, bin_ws.data_ptr(), ws.data_ptr(), ws_bytes, img.data_ptr(),
                                    con.data_ptr(), ft.data_ptr(), rg.data_ptr(), gsid.data_ptr(), st)

    ok = [aligned_empty((3, Hi, Wi)), aligned_empty((Hi, Wi), torch.int32), aligned_empty((Hi, Wi)),
          aligned_empty((T, 2), torch.int32)]
    assert render(*ok) == 0
    torch.cuda.synchronize()
    for i, dt in enumerate((torch.float32, torch.int32, torch.float32, torch.int32)):
        args = list(ok)
        args[i] = shifted_empty(tuple(ok[i].shape), dt)
        rc = render(*args)
        assert rc != 0 and b"misaligned" in lib.gsb_last_error(), i
