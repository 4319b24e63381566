"""GPU parity for SURVEY 8f row N3: density control and Gaussian record conversion through the
C ABI, against oracle/density_oracle.py (pinned to the reference by test_oracle_density.py)
and directly against the reference's own outputs in tests/golden/density.npz / gsio.npz.

Index work (classes, slots, counts, which row lands where, moved rows) is bit exact;
recomputed values (logit o sigmoid, log o exp, normalise, split offsets) agree to 3e-6
relative -- the ulp-level spread between libdevice and glibc/torch-CPU expf/logf."""
import os

import numpy as np
import pytest
import torch

from oracle import density_oracle as do

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = "cuda"
NAMES = do.NAMES


def t(a, dtype=None):
    x = torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    return x.to(dtype) if dtype is not None else x


def n(x):
    return x.detach().cpu().numpy()


def close(got, want, name, rtol=3e-6, atol=2e-6):
    assert got.shape == want.shape, (name, got.shape, want.shape)
    fin = np.isfinite(want)
    assert np.array_equal(np.isfinite(got), fin), name
    assert np.array_equal(got[~fin], want[~fin]), name
    err = np.abs(got[fin].astype(np.float64) - want[fin]) - (rtol * np.abs(want[fin]) + atol)
    assert (err <= 0).all(), "%s: max excess %.3e" % (name, err.max())


@pytest.fixture(scope="module")
def dens():
    return dict(np.load(os.path.join(G, "density.npz")))


@pytest.fixture(scope="module")
def gsio():
    return dict(np.load(os.path.join(G, "gsio.npz")))


def make_adam(params):
    from easygaussiansplatting_b200.gau_io import adam_groups
    return torch.optim.Adam(adam_groups(params), lr=0.0, eps=1e-15)


@pytest.mark.parametrize("tag", ["s_", "n_"])
def test_controller_matches_reference_fixture(dens, tag):
    """the whole GSModel density API on a real torch.optim.Adam, against what the reference's
    gsmodel.py produced for the same inputs and the same unit normals"""
    from easygaussiansplatting_b200.density import DensityController
    has_state = (tag + "in_m_pws") in dens
    params = {k: t(dens[tag + "in_" + k]).requires_grad_() for k in NAMES}
    opt = make_adam(params)
    if has_state:
        for g in opt.param_groups:
            p = g["params"][0]
            opt.state[p] = {"step": torch.tensor(1.0), "exp_avg": t(dens[tag + "in_m_" + g["name"]]),
                            "exp_avg_sq": t(dens[tag + "in_v_" + g["name"]])}
    ctl = DensityController(float(dens[tag + "sense_size"]), verbose=False)
    for it in range(3):
        ctl.update_density_info(t(dens[tag + "acc%d_dloss_dus" % it]), t(dens[tag + "acc%d_mask" % it]))
        close(n(ctl.grad_accum), dens[tag + "acc%d_grad_accum" % it], "grad_accum %d" % it, rtol=1e-6, atol=1e-13)
        assert np.array_equal(n(ctl.cunt), dens[tag + "acc%d_cunt" % it])

    z = t(dens[tag + "z"])   # hand the fixture's unit normals to the controller
    orig = torch.Tensor.normal_
    torch.Tensor.normal_ = lambda self, *a, **k: self.copy_(z) if self.shape == z.shape else orig(self, *a, **k)
    try:
        rep = ctl.update_gaussian_density(params, opt)
    finally:
        torch.Tensor.normal_ = orig
    Nin, Nout = dens[tag + "in_pws"].shape[0], dens[tag + "out_pws"].shape[0]
    assert rep["total"] == Nout and rep["splited"] == z.shape[0] and rep["pruned"] == Nin - (Nout - rep["cloned"] - rep["splited"])
    K = Nout - rep["cloned"] - rep["splited"]
    assert ctl.grad_accum is None and ctl.cunt is None
    for g in opt.param_groups:
        k, p = g["name"], g["params"][0]
        assert params[k] is p and p.requires_grad and p.is_leaf
        assert np.array_equal(n(p)[:K], dens[tag + "out_" + k][:K]), k          # moved rows: bit exact
        close(n(p), dens[tag + "out_" + k], "out " + k)
        st = opt.state.get(p, None)
        if has_state:
            assert np.array_equal(n(st["exp_avg"]), dens[tag + "out_m_" + k]), k
            assert np.array_equal(n(st["exp_avg_sq"]), dens[tag + "out_v_" + k]), k
        else:
            assert st is None or "exp_avg" not in st
    assert len(opt.state) == (6 if has_state else 0)
    # the rebuilt optimizer must still step
    for g in opt.param_groups:
        g["params"][0].grad = torch.ones_like(g["params"][0])
        g["lr"] = 1e-3
    opt.step()
    assert all(opt.state[g["params"][0]]["exp_avg"].shape == g["params"][0].shape for g in opt.param_groups)
    if has_state:
        # reset_alpha on a fresh copy of the fixture's post-update state
        params2 = {k: t(dens[tag + "out_" + k]).requires_grad_() for k in NAMES}
        opt2 = make_adam(params2)
        pa = params2["alphas_raw"]
        opt2.state[pa] = {"step": torch.tensor(1.0), "exp_avg": t(dens[tag + "out_m_alphas_raw"]),
                          "exp_avg_sq": t(dens[tag + "out_v_alphas_raw"])}
        ctl.reset_alpha(params2, opt2)
        close(n(pa), dens[tag + "reset_alphas_raw"], "reset", rtol=1e-6, atol=0)
        assert not n(opt2.state[pa]["exp_avg"]).any() and not n(opt2.state[pa]["exp_avg_sq"]).any()


def random_state(N, seed, sense=5.0):
    rng = np.random.default_rng(seed)
    P = dict(pws=rng.uniform(-2, 2, (N, 3)), low_shs=rng.normal(size=(N, 3)), high_shs=rng.normal(size=(N, 45)) * 0.1,
             alphas_raw=rng.uniform(-7.5, 4, (N, 1)),
             scales_raw=np.log(np.exp(rng.uniform(np.log(0.002 * sense), np.log(0.12 * sense), (N, 1))) *
                               rng.uniform(0.6, 1.5, (N, 3))),
             rots_raw=rng.normal(size=(N, 4)) * rng.uniform(0.3, 2, (N, 1)))
    P = {k: v.astype(np.float32) for k, v in P.items()}
    M = {k: (rng.normal(size=v.shape) * 1e-3).astype(np.float32) for k, v in P.items()}
    V = {k: (rng.uniform(size=v.shape) * 1e-6).astype(np.float32) for k, v in P.items()}
    acc = (np.abs(rng.normal(size=(N, 1))) * 1.5e-6).astype(np.float32)
    cnt = rng.integers(0, 6, N).astype(np.int32)
    acc[cnt == 0] = 0
    return P, M, V, acc, cnt


@pytest.mark.parametrize("N,seed", [(1, 1), (257, 2), (50000, 3)])
def test_plan_and_apply_vs_oracle(N, seed):
    from easygaussiansplatting_b200 import density
    P, M, V, acc, cnt = random_state(N, seed)
    th_o = do.thresholds(5.0)
    th = density.raw_thresholds(5.0)
    cls_o = do.classify(P["alphas_raw"], P["scales_raw"], acc, cnt, th_o)
    dP = {k: t(v) for k, v in P.items()}
    cls, slots, counts = density.plan(dP["alphas_raw"], dP["scales_raw"], t(acc), t(cnt), th)
    assert np.array_equal(n(cls), cls_o)
    flags = np.stack([cls_o != do.PRUNE, cls_o == do.CLONE, cls_o == do.SPLIT], axis=1).astype(np.int64)
    assert np.array_equal(n(slots), np.cumsum(flags, axis=0) - flags)
    assert counts == tuple(int(x) for x in flags.sum(axis=0))
    z = np.random.default_rng(seed + 100).normal(size=(counts[2], 3)).astype(np.float32)
    oP, oM, oV, ocounts = do.densify(P, M, V, cls_o, z)
    assert ocounts == counts
    dst, dm, dv = density.apply(cls, slots, counts, dP, {k: t(v) for k, v in M.items()}, {k: t(v) for k, v in V.items()}, t(z))
    K = counts[0]
    for k in NAMES:
        assert np.array_equal(n(dst[k])[:K], oP[k][:K]), k
        close(n(dst[k]), oP[k], k)
        assert np.array_equal(n(dm[k]), oM[k]) and np.array_equal(n(dv[k]), oV[k]), k
    # without optimizer state
    dst2, dm2, dv2 = density.apply(cls, slots, counts, dP, None, None, t(z))
    assert dm2 is None and dv2 is None
    for k in NAMES:
        assert torch.equal(dst2[k], dst[k])


def random_state_device(N, seed, sense=5.0):
    """random_state's distribution, drawn on the GPU from a seeded torch.Generator"""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    U = lambda shape, a, b: torch.empty(shape, device=DEV).uniform_(a, b, generator=gen)
    Nn = lambda shape, s=1.0: torch.empty(shape, device=DEV).normal_(0.0, s, generator=gen)
    scale = U((N, 1), np.log(0.002 * sense), np.log(0.12 * sense)).exp_() * U((N, 3), 0.6, 1.5)
    P = dict(pws=U((N, 3), -2, 2), low_shs=Nn((N, 3)), high_shs=Nn((N, 45), 0.1), alphas_raw=U((N, 1), -7.5, 4),
             scales_raw=scale.log_(), rots_raw=Nn((N, 4)).mul_(U((N, 1), 0.3, 2)))
    M = {k: Nn(v.shape, 1e-3) for k, v in P.items()}
    V = {k: U(v.shape, 0.0, 1e-6) for k, v in P.items()}
    cnt = torch.randint(0, 6, (N,), device=DEV, generator=gen, dtype=torch.int32)
    acc = Nn((N, 1), 1.5e-6).abs_().mul_((cnt > 0).unsqueeze(1))
    return P, M, V, acc, cnt


def test_apply_64bit_kernel_equals_row_group_slices():
    """N = 23 000 037 takes the row-group kernel with 64-bit destination offsets (all 18 parameter
    / Adam-moment jobs, element offsets past 1e9 in high_shs); two row slices below 23 M take its
    32-bit instantiation.  Classification is per row and slots are prefix sums, so each output row
    of the full run has a known place in one slice's output: kept row k of slice 2 is full row
    K1 + k, its clones K + C1 + c, its splits K + C + S1 + s.  All rows must be bit-identical."""
    from easygaussiansplatting_b200 import density
    N, N1 = 23_000_037, 11_500_011
    need = 44 << 30
    free, total = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB of %.1f GB free" % (need / 2**30, free / 2**30,
                                                                                    total / 2**30))
    torch.cuda.reset_peak_memory_stats()
    P, M, V, acc, cnt = random_state_device(N, 23)
    th = density.raw_thresholds(5.0)
    cls, slots, (K, Cn, S) = density.plan(P["alphas_raw"], P["scales_raw"], acc, cnt, th)
    assert K > 0 and Cn > 0 and S > 0 and 0.9 * N < K + Cn + S < 1.1 * N, (K, Cn, S)
    z = torch.randn((S, 3), device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    full = density.apply(cls, slots, (K, Cn, S), P, M, V, z)
    sl = lambda d, a, b: {k: v[a:b] for k, v in d.items()}
    c_done = s_done = 0
    for a, b in ((0, N1), (N1, N)):
        cls_i, slots_i, (Ki, Ci, Si) = density.plan(P["alphas_raw"][a:b], P["scales_raw"][a:b], acc[a:b], cnt[a:b],
                                                   th)
        assert torch.equal(cls_i, cls[a:b])
        k_done = 0 if a == 0 else K - Ki
        part = density.apply(cls_i, slots_i, (Ki, Ci, Si), sl(P, a, b), sl(M, a, b), sl(V, a, b),
                             z[s_done:s_done + Si])
        for d_full, d_part, what in zip(full, part, ("param", "exp_avg", "exp_avg_sq")):
            for k in NAMES:
                f, p = d_full[k], d_part[k]
                assert torch.equal(f[k_done:k_done + Ki], p[:Ki]), (a, what, k, "kept")
                assert torch.equal(f[K + c_done:K + c_done + Ci], p[Ki:Ki + Ci]), (a, what, k, "cloned")
                assert torch.equal(f[K + Cn + s_done:K + Cn + s_done + Si], p[Ki + Ci:]), (a, what, k, "split")
        c_done, s_done = c_done + Ci, s_done + Si
        del part, cls_i, slots_i
        torch.cuda.empty_cache()
    assert c_done == Cn and s_done == S
    print("N %d: K %d C %d S %d, peak device memory %.2f GB" % (N, K, Cn, S,
                                                                  torch.cuda.max_memory_allocated() / 2**30))


def test_degenerate_populations():
    """everything pruned / nothing selected / N = 0"""
    from easygaussiansplatting_b200 import density
    P, M, V, acc, cnt = random_state(300, 9)
    th = density.raw_thresholds(5.0)
    dP = {k: t(v) for k, v in P.items()}
    allp = dict(th, alpha_raw_min=1e9)
    cls, slots, counts = density.plan(dP["alphas_raw"], dP["scales_raw"], t(acc), t(cnt), allp)
    assert counts == (0, 0, 0) and (n(cls) == 3).all()
    dst, _, _ = density.apply(cls, slots, counts, dP, None, None, torch.empty((0, 3), device=DEV))
    assert all(v.shape[0] == 0 for v in dst.values())
    none = dict(th, grad_min=1e9, alpha_raw_min=-1e9, scale_raw_max=1e9)
    cls, slots, counts = density.plan(dP["alphas_raw"], dP["scales_raw"], t(acc), t(cnt), none)
    assert counts == (300, 0, 0)
    dst, _, _ = density.apply(cls, slots, counts, dP, None, None, torch.empty((0, 3), device=DEV))
    assert all(torch.equal(dst[k], dP[k]) for k in NAMES)
    e = {k: torch.empty((0, w), device=DEV) for k, w in zip(NAMES, (3, 3, 45, 1, 3, 4))}
    cls, slots, counts = density.plan(e["alphas_raw"], e["scales_raw"], torch.empty((0, 1), device=DEV),
                                      torch.empty(0, dtype=torch.int32, device=DEV), th)
    assert counts == (0, 0, 0)


def test_full_size_properties():
    """1M Gaussians: the rebuilt tensors equal torch's own boolean gathers of the inputs
    (survivors, clone sources, split sources), and every recomputed column is an involution
    fixed point: applying the clone transform twice changes nothing beyond 1 ulp"""
    from easygaussiansplatting_b200 import density
    N = 1_000_000
    P, M, V, acc, cnt = random_state(N, 5)
    dP, dM, dV = ({k: t(v) for k, v in X.items()} for X in (P, M, V))
    th = density.raw_thresholds(5.0)
    cls, slots, (K, Cn, S) = density.plan(dP["alphas_raw"], dP["scales_raw"], t(acc), t(cnt), th)
    assert K + Cn + S > N // 2 and Cn > 1000 and S > 1000 and K < N
    z = torch.randn((S, 3), device=DEV)
    dst, dm, dv = density.apply(cls, slots, (K, Cn, S), dP, dM, dV, z)
    keep, cl, sp = cls != 3, cls == 1, cls == 2
    for k in NAMES:
        assert torch.equal(dst[k][:K], dP[k][keep]), k
        assert torch.equal(dm[k][:K], dM[k][keep]) and torch.equal(dv[k][:K], dV[k][keep]), k
        assert not dm[k][K:].any() and not dv[k][K:].any(), k
    for k in ("low_shs", "high_shs"):
        assert torch.equal(dst[k][K:K + Cn], dP[k][cl]) and torch.equal(dst[k][K + Cn:], dP[k][sp]), k
    assert torch.equal(dst["pws"][K:K + Cn], dP["pws"][cl])
    # split offsets: |offset| = |z * 0.6^-1 * new_scale| because R(q) is a rotation
    off = dst["pws"][K + Cn:] - dP["pws"][sp]
    want = (z * torch.exp(dst["scales_raw"][K + Cn:]) / 0.6).norm(dim=1)
    assert torch.allclose(off.norm(dim=1), want, rtol=2e-4, atol=1e-6)
    assert torch.allclose(dst["scales_raw"][K + Cn:], dP["scales_raw"][sp] + np.log(0.6), atol=2e-6)
    assert torch.allclose(dst["rots_raw"][K:].norm(dim=1), torch.ones(Cn + S, device=DEV), atol=1e-6)
    assert torch.allclose(torch.sigmoid(dst["alphas_raw"][K:]), torch.sigmoid(torch.cat([dP["alphas_raw"][cl], dP["alphas_raw"][sp]])),
                          atol=1e-6)


@pytest.mark.parametrize("tag", ["deg3", "deg1"])
def test_gau_io_matches_reference_fixture(gsio, tag, tmp_path):
    from easygaussiansplatting_b200 import gau_io
    p = str(tmp_path / "scene.ply")
    open(p, "wb").write(gsio[tag + "_ply"].tobytes())
    gs = gau_io.load_ply(p)
    assert gs.dtype == np.dtype(gau_io.gsdata_type(gsio[tag + "_sh"].shape[1]))
    for k in ("pw", "sh"):
        assert np.array_equal(np.asarray(gs[k]), gsio[tag + "_" + k]), k
    for k in ("rot", "scale", "alpha"):
        close(np.asarray(gs[k]), gsio[tag + "_" + k], k, rtol=2e-6, atol=1e-7)
    # recarray -> training tensors (get_training_params), from the REFERENCE's recarray
    ref_gs = np.zeros(len(gs), dtype=gs.dtype)
    for k in ("pw", "rot", "scale", "alpha", "sh"):
        ref_gs[k] = gsio[tag + "_" + k]
    params, groups = gau_io.get_training_params(ref_gs)
    assert [g["name"] for g in groups] == list(NAMES) and groups[2]["lr"] == 0.001 / 20
    for k in NAMES:
        assert params[k].requires_grad and params[k].is_leaf
        close(n(params[k]), gsio[tag + "_tp_" + k], "training " + k)
    assert np.array_equal(n(params["high_shs"]), gsio[tag + "_tp_high_shs"])
    # training tensors -> .npy (save_training_params), from the REFERENCE's tensors
    ref_params = {k: t(gsio[tag + "_tp_" + k]) for k in NAMES}
    fn = str(tmp_path / "out.npy")
    gau_io.save_training_params(fn, ref_params)
    back = gau_io.load_gs(fn)
    assert back.dtype == np.dtype(gau_io.gsdata_type(48))
    for k in ("pw", "rot", "scale", "alpha", "sh"):
        close(np.asarray(back[k]), gsio[tag + "_back_" + k], "saved " + k, rtol=3e-6, atol=1e-7)
    # disk -> device without the host round trip, and save_ply -> load_ply closes the loop
    p2, _ = gau_io.load_training_params(p)
    for k in NAMES:
        close(n(p2[k]), gsio[tag + "_tp_" + k], "direct " + k, rtol=5e-6, atol=3e-6)
    q = str(tmp_path / "again.ply")
    gau_io.save_ply(q, gs)
    again = gau_io.load_ply(q)
    for k in ("pw", "rot", "scale", "alpha", "sh"):
        close(np.asarray(again[k]), np.asarray(gs[k]), "round trip " + k, rtol=3e-6, atol=1e-7)


def test_gau_io_full_size_round_trip(tmp_path):
    """1M-Gaussian SH-3 checkpoint (248 MB): params -> gs rows -> save_ply -> load -> params
    returns the starting tensors (to the float32 round trip of exp/log/sigmoid/logit)"""
    from easygaussiansplatting_b200 import gau_io
    N = 1_000_000
    P, _, _, _, _ = random_state(N, 8)
    P["alphas_raw"] = np.clip(P["alphas_raw"], -6, 4)
    dP = {k: t(v) for k, v in P.items()}
    rows = gau_io.params_to_gs_rows(dP)
    assert rows.shape == (N, 59)
    gs = gau_io._rows_to_recarray(rows, 48)
    p = str(tmp_path / "big.ply")
    gau_io.save_ply(p, gs)
    back, _ = gau_io.load_training_params(p)
    for k in ("pws", "low_shs", "high_shs"):
        assert torch.equal(back[k].detach(), dP[k]), k
    assert torch.allclose(back["scales_raw"].detach(), dP["scales_raw"], atol=3e-6)
    assert torch.allclose(back["alphas_raw"].detach(), dP["alphas_raw"], rtol=2e-5, atol=2e-5)
    nrm = dP["rots_raw"] / dP["rots_raw"].norm(dim=1, keepdim=True)
    assert torch.allclose(back["rots_raw"].detach(), nrm, atol=1e-6)
