"""CPU checks of MCMC densification: the oracle's relocation series against numerical integration,
its opacity and r = 1 identities, the integer sampler's frequencies, the row order and moment
zeroing of relocate and grow on hand-built cases, and the C ABI / sm_90a binary of the kernels."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest
from scipy import integrate, stats

from oracle import mcmc_oracle as omc

from test_host_cpu import header_symbols

F = np.float32
OPACITIES = (0.005, 0.01, 0.1, 0.37, 0.5, 0.8, 0.99, 0.999999, 1 - 2.0 ** -23)


def _integral(op, r):
    """int (1 - (1 - op e^(-x^2/2))^r) dx / sqrt(2 pi), the footprint of r copies of opacity op"""
    f = lambda x: -np.expm1(r * np.log1p(-op * np.exp(-0.5 * x * x)))  # noqa: E731
    v, _ = integrate.quad(f, -np.inf, np.inf, epsabs=0, epsrel=1e-13, limit=400)
    return v / np.sqrt(2 * np.pi)


def test_series_equals_the_footprint_integral():
    worst = 0.0
    for r in range(1, 52):
        for o in OPACITIES:
            op, _ = omc.new_opacity(o, 1 - omc.L(o), r)
            got = float(omc.series(op, r))
            want = _integral(float(op), r)
            worst = max(worst, abs(got - want) / want)
    assert worst <= 1e-10, worst


def test_new_opacity_keeps_the_transmittance_and_r1_is_the_identity():
    for r in range(1, 52):
        for o in OPACITIES:
            op, q = omc.new_opacity(o, 1 - omc.L(o), r)
            if omc.L(0.005) < op < omc.L(1) - omc.L(2) ** -23:  # unclamped
                assert abs(q ** r - (1 - omc.L(o))) <= 1e-15 and abs(op + q - 1) <= 1e-18, (o, r)
    rng = np.random.default_rng(0)
    for a in rng.uniform(-5, 15, size=50).astype(F):  # o inside the clamp range
        o, om = (omc.L(1) / (omc.L(1) + np.exp(x)) for x in (-omc.L(float(a)), omc.L(float(a))))
        assert omc.new_opacity(o, om, 1) == (o, om) and omc.series(o, 1) == o
        s = rng.normal(size=3).astype(F)
        a1, s1 = omc.relocation_value(a, s, 0, n_max=51)  # c = 0 hits: r = 1
        assert np.array_equal(s1, s)  # scale factor exactly 1
        assert abs(float(a1) - float(a)) <= 2 * float(np.spacing(np.abs(a)))


def test_fp32_series_loses_its_digits_at_r51():
    """the reason the kernels evaluate the series in fp64: in fp32 the alternating sum at r = 51 and
    o near 1 is off by far more than an fp32 ulp of the result"""
    op, _ = omc.new_opacity(1 - 2.0 ** -23, 2.0 ** -23, 51)
    exact = float(omc.series(op, 51))
    s, binom, p = F(0), F(1), F(1)
    for m in range(1, 52):
        binom = F(binom * F(51 - m + 1) / F(m))
        p = F(p * F(op))
        t = F(binom * p / F(np.sqrt(F(m))))
        s = F(s + t) if m % 2 else F(s - t)
    assert abs(float(s) - exact) / exact > 100 * 2.0 ** -23  # hundreds of fp32 ulps


def test_integer_sampler_frequencies_match_the_weights():
    rng = np.random.default_rng(5)
    a = rng.normal(size=40).astype(F) * 3
    a[[3, 17]] = np.nan
    a[[5, 9]] = -8.0  # dead in relocate, tiny weight in grow
    for mode in ("relocate", "grow"):
        w = omc.weights(a, mode)
        assert w[3] == 0 and w[17] == 0 and bool((w[[5, 9]] == 0).all()) == (mode == "relocate")
        u = rng.random(400000)
        ids = omc.sample(w, u)
        assert not np.isin(ids, np.flatnonzero(w == 0)).any()
        obs = np.bincount(ids, minlength=len(a))
        keep = w > 0
        exp = w[keep].astype(np.float64) / float(w.sum(dtype=np.uint64)) * len(u)
        big = exp >= 5
        chi = stats.chisquare(obs[keep][big], exp[big] * obs[keep][big].sum() / exp[big].sum())
        assert chi.pvalue > 1e-3, (mode, chi)
    # boundaries: u = 0 is the first weighted row, u -> 1 the last
    w = np.array([0, 3, 0, 5, 0], np.uint64)
    assert omc.sample(w, np.array([0.0, np.nextafter(1.0, 0), 3 / 8 - 1e-12, 3 / 8])).tolist() == [1, 3, 1, 3]


def _params(N, seed, D=0):
    rng = np.random.default_rng(seed)
    p = {k: rng.normal(size=(N, w)).astype(F) for k, w in omc.dor.WIDTH.items()}
    if D:
        p["features"] = rng.normal(size=(N, D)).astype(F)
    return p


def test_relocate_row_order_and_moments():
    N = 8
    p = _params(N, 1, D=3)
    p["alphas_raw"][:, 0] = [2.0, -9.0, 0.5, np.nan, 1.0, -6.0, 3.0, -9.5]
    m = {k: np.ones_like(x) for k, x in p.items()}
    v = {k: 2 * np.ones_like(x) for k, x in p.items()}
    u = np.array([0.01, 0.5, 0.99, 0.7])
    out, mo, vo, dead, sampled = omc.relocate(p, m, v, u)
    assert dead.tolist() == [1, 3, 5, 7]  # ascending, NaN included
    assert not np.isin(sampled, dead).any()
    for j, (d, s) in enumerate(zip(dead, sampled)):
        for k in out:
            assert np.array_equal(out[k][d], out[k][s]), k
    hit = np.unique(sampled)
    for i in range(N):
        if i in hit:
            c = int((sampled == i).sum())
            a, s = omc.relocation_value(p["alphas_raw"][i, 0], p["scales_raw"][i], c)
            assert out["alphas_raw"][i, 0] == a and np.array_equal(out["scales_raw"][i], s)
            assert F(1) / (F(1) + np.exp(-a)) < F(1) / (F(1) + np.exp(-p["alphas_raw"][i, 0]))
        elif i not in dead:
            for k in out:
                assert np.array_equal(out[k][i], p[k][i]), k
    for d in (mo, vo):
        for k in d:
            zero = np.zeros(N, bool)
            zero[dead] = zero[sampled] = True
            assert not d[k][zero].any() and (d[k][~zero] != 0).all(), k
    # no state: moments stay None; nothing alive: a no-op
    assert omc.relocate(p, None, None, u)[1] is None
    q = _params(4, 2)
    q["alphas_raw"][:] = -20.0
    out, _, _, dead, sampled = omc.relocate(q, None, None, np.zeros(4))
    assert len(sampled) == 0 and out is q


def test_grow_row_order_and_moments():
    N = 6
    p = _params(N, 3, D=2)
    p["alphas_raw"][:, 0] = [0.0, np.nan, 4.0, -3.0, 1.0, -9.0]
    m = {k: np.ones_like(x) for k, x in p.items()}
    v = {k: np.ones_like(x) for k, x in p.items()}
    assert omc.grow_count(N, 100, 0.5) == 3 and omc.grow_count(N, 7, 0.5) == 1
    assert omc.grow_count(19, 100) == 0 and omc.grow_count(100, 50) == 0
    out, mo, vo, sampled = omc.grow(p, m, v, np.array([0.05, 0.5, 0.95]), 3)
    assert 1 not in sampled.tolist()  # a NaN row is never a source
    for k in out:
        assert out[k].shape[0] == N + 3
        assert np.array_equal(out[k][N:], out[k][sampled]), k
        for i in range(N):
            if i not in sampled and k not in ("alphas_raw", "scales_raw"):
                assert np.array_equal(out[k][i], p[k][i], equal_nan=True)
    for d in (mo, vo):
        for k in d:
            zero = np.zeros(N + 3, bool)
            zero[N:] = zero[sampled] = True
            assert not d[k][zero].any() and (d[k][~zero] == 1).all(), k


def test_noise_oracle_is_sigma_z():
    rng = np.random.default_rng(4)
    N = 30
    p = _params(N, 6)
    z = rng.normal(size=(N, 3))
    d = omc.noise(p, z, 1e-3)
    for i in range(N):
        q = p["rots_raw"][i].astype(np.float64)
        q = q / np.linalg.norm(q)
        R = omc.dor._rotate(q[None].astype(F), np.eye(3, dtype=F)).T.astype(np.float64)  # columns R e_j
        S = R @ np.diag(np.exp(2 * p["scales_raw"][i].astype(np.float64))) @ R.T
        o = 1 / (1 + np.exp(-float(p["alphas_raw"][i, 0])))
        g = 1 / (1 + np.exp(-100 * ((1 - o) - 0.995)))
        assert np.allclose(d[i], S @ z[i] * 1e-3 * 5e5 * g, rtol=1e-5, atol=0)


# ---------------------------------------------------------------- the C ABI and the sm_90a binary
MCMC_SYMBOLS = ("gsb_mcmc_workspace_bytes", "gsb_mcmc_plan", "gsb_mcmc_sample", "gsb_mcmc_relocate",
                "gsb_mcmc_relocate_rows", "gsb_mcmc_grow", "gsb_mcmc_grow_rows", "gsb_mcmc_noise")


def test_mcmc_symbols_signatures_and_workspace_queries():
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    lib = _lib.load()
    syms = header_symbols()
    for s in MCMC_SYMBOLS:
        assert s in syms and s in _lib.SIGNATURES and hasattr(lib, s), s
    prev = 0
    for N in (0, 1, 1000, 1 << 20, 5 << 20):
        b = lib.gsb_mcmc_workspace_bytes(N, N)
        assert b >= 256 + 32 * N and b >= prev and b % 256 == 0
        assert lib.gsb_mcmc_workspace_bytes(N, N + 1000) >= b + 16 * 1000 - 256
        prev = b
    vp = C.c_void_p
    counts = (C.c_int64 * 2)(7, 7)
    assert lib.gsb_mcmc_plan(0, None, F(0), 0, None, 0, counts, None) == 0 and list(counts) == [0, 0]
    assert lib.gsb_mcmc_plan(10, vp(16), F(0), 2, vp(256), 1 << 20, counts, None) != 0
    assert b"mode" in lib.gsb_last_error()
    assert lib.gsb_mcmc_plan(10, vp(16), F(0), 0, vp(264), 1 << 20, counts, None) != 0
    assert b"misaligned" in lib.gsb_last_error()
    assert lib.gsb_mcmc_plan(10, vp(16), F(0), 0, vp(256), 64, counts, None) != 0
    assert b"too small" in lib.gsb_last_error()
    assert lib.gsb_mcmc_relocate(10, 11, vp(16), vp(256), 1 << 20, 0.005, 51, None, None, None, None) != 0
    assert b"bad counts" in lib.gsb_last_error()
    assert lib.gsb_mcmc_relocate(10, 2, vp(16), vp(256), 1 << 20, 0.005, 52, None, None, None, None) != 0
    assert b"n_max" in lib.gsb_last_error()
    assert lib.gsb_mcmc_sample(0, 3, vp(16), vp(256), 1 << 20, vp(16), None) != 0
    assert lib.gsb_mcmc_grow_rows(0, 0, None, None, 0, 4, None, None, None, None, None, None, None) == 0
    assert lib.gsb_mcmc_noise(0, None, None, None, None, None, F(1), F(100), F(0.995), None) == 0


def test_mcmc_kernels_are_sm90a_without_spills():
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    kernels = ("k_mcmc_weight_count", "k_mcmc_scan_blocks", "k_mcmc_prefix", "k_mcmc_sample", "k_mcmc_values",
               "k_mcmc_relocate", "k_mcmc_relocate_rows", "k_mcmc_grow_copy", "k_mcmc_grow_append",
               "k_mcmc_grow_rows", "k_mcmc_noise")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert set(re.findall(r"code for (sm_\w+)", sass)) == {"sm_90a"}
    funcs = re.split(r"\n\s*Function : ", sass)
    for name in kernels:
        body = [f for f in funcs if re.match(r"\S*%d%sE" % (len(name), name), f)]
        assert len(body) == 1, name
    # the relocation value is fp64 arithmetic (the reason for DESIGN 3.11's precision note)
    values = [f for f in funcs if re.match(r"\S*13k_mcmc_valuesE", f)][0]
    assert "DFMA" in values or "DMUL" in values
    r = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True)
    found = re.findall(r"Function (\S*k_mcmc_\w*):\s*\n\s*(REG:.*)", r.stdout)
    assert sorted(set(re.sub(r"^\S*?\d+(k_mcmc_[a-z_]+)E.*$", r"\1", f) for f, _ in found)) == sorted(kernels)
    for name, usage in found:
        assert "LOCAL:0 " in usage and "STACK:0 " in usage, (name, usage)
    lib = _lib.load()
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    for k in ("mcmc_scan", "mcmc_sample", "mcmc_relocate", "mcmc_grow", "mcmc_rows", "mcmc_noise"):
        assert k in names, k
    assert names[-2:] == ["draw_rgbd", "draw_backward_rgbd"]
