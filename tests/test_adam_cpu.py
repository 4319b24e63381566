"""CPU checks of the fused Adam step: the fp64 oracle against torch.optim.Adam in float64, its
selective rule on hand-built cases, the C ABI (symbols, argument errors, no-op cases) and the sm_90a
binary of the kernel."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import adam_oracle as oad

from test_host_cpu import header_symbols


# ---------------------------------------------------------------- the oracle
@pytest.mark.parametrize("betas,eps", [((0.9, 0.999), 1e-8), ((0.9, 0.999), 1e-15), ((0.3, 0.5), 1e-3),
                                       ((0.0, 0.99), 1e-8)])
def test_oracle_equals_torch_adam_in_float64(betas, eps):
    rng = np.random.default_rng(0)
    shapes = [(17, 3), (17, 45), (17, 1), (5, 7)]
    lrs = [1e-3, 2.5e-2, 0.0, 0.1]
    ps = [torch.nn.Parameter(torch.from_numpy(rng.normal(size=s))) for s in shapes]
    opt = torch.optim.Adam([{"params": [p], "lr": lr} for p, lr in zip(ps, lrs)], betas=betas, eps=eps,
                           foreach=False)
    ref = [(p.detach().numpy().copy(), np.zeros(s), np.zeros(s), 0) for p, s in zip(ps, shapes)]
    for _ in range(20):
        gs = [rng.normal(size=s) * rng.choice([1e-4, 1.0, 30.0]) for s in shapes]
        for p, g in zip(ps, gs):
            p.grad = torch.from_numpy(g)
        opt.step()
        ref = [oad.adam_step(pp, g, mm, vv, tt, lr, *betas, eps) for (pp, mm, vv, tt), g, lr in zip(ref, gs, lrs)]
    for p, (pp, mm, vv, tt) in zip(ps, ref):
        st = opt.state[p]
        assert float(st["step"]) == tt == 20
        for got, want in ((p.detach().numpy(), pp), (st["exp_avg"].numpy(), mm), (st["exp_avg_sq"].numpy(), vv)):
            np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-300)


def test_oracle_adam_step_argument_order():
    # adam_step(p, g, m, v, t, ...) with t the count before the step
    p, g, m, v = np.ones(2), np.array([1.0, -2.0]), np.zeros(2), np.zeros(2)
    p1, m1, v1, t1 = oad.adam_step(p, g, m, v, 0, 0.1)
    assert t1 == 1
    # the first step of Adam moves every coordinate by about lr against the sign of its gradient
    np.testing.assert_allclose(p1, [0.9, 1.1], rtol=1e-6)
    np.testing.assert_allclose(m1, 0.1 * g)
    np.testing.assert_allclose(v1, 0.001 * g * g)


def test_oracle_selective_rule():
    rng = np.random.default_rng(1)
    N, D = 6, 3
    p, m, v = rng.normal(size=(N, D)), rng.normal(size=(N, D)), rng.random((N, D))
    g = rng.normal(size=(N, D))
    vis = np.array([1, 0, 0, 1, 1, 0], bool)
    pn, mn, vn, t = oad.adam_step(p, g, m, v, 4, 1e-2, visibility=vis)
    assert t == 5  # the step count advances whatever the mask
    for new, old in ((pn, p), (mn, m), (vn, v)):
        assert np.array_equal(new[~vis], old[~vis])  # invisible rows: exactly the inputs
    pd, md, vd, _ = oad.adam_step(p, g, m, v, 4, 1e-2)
    for new, dense in ((pn, pd), (mn, md), (vn, vd)):
        assert np.array_equal(new[vis], dense[vis])  # visible rows: the dense update at the same t
    # all-false: nothing changes but t; all-true: the dense step
    pz, mz, vz, tz = oad.adam_step(p, g, m, v, 4, 1e-2, visibility=np.zeros(N, bool))
    assert tz == 5 and np.array_equal(pz, p) and np.array_equal(mz, m) and np.array_equal(vz, v)
    pa, _, _, _ = oad.adam_step(p, g, m, v, 4, 1e-2, visibility=np.ones(N, bool))
    assert np.array_equal(pa, pd)


# ---------------------------------------------------------------- the C ABI and the sm_90a binary
def _lib():
    from easygaussiansplatting_b200 import _lib, build
    build.build()
    return _lib, _lib.load()


def test_adam_symbol_and_table_layout():
    L, lib = _lib()
    assert "gsb_adam_step" in header_symbols() and "gsb_adam_step" in L.SIGNATURES and hasattr(lib, "gsb_adam_step")
    # gsb_adam_tensor: four pointers, int64 numel, int32 D, two floats (56 bytes with padding)
    assert C.sizeof(L.AdamTensor) == 56
    assert [f for f, _ in L.AdamTensor._fields_] == ["param", "grad", "exp_avg", "exp_avg_sq", "numel", "D",
                                                      "step_size", "bc2_sqrt"]


def test_adam_argument_errors_and_no_ops():
    L, lib = _lib()
    T = L.AdamTensor
    vp = C.c_void_p

    def call(rows, N=0, vis=None, b1=0.9, b2=0.999, eps=1e-8, n=None):
        table = (T * max(len(rows), 1))(*rows)
        return lib.gsb_adam_step(len(rows) if n is None else n, table if rows or n else None, N, vp(vis), b1, b2,
                                 eps, None)

    good = lambda numel, D=0: T(16, 32, 48, 64, numel, D, 1e-3, 0.5)  # noqa: E731
    # no-ops: an empty table, N = 0, zero-element tensors (no device needed: nothing is launched)
    assert call([]) == 0
    assert call([], N=0, vis=256) == 0
    assert call([good(0, 3)], N=0, vis=256) == 0
    assert call([T(None, None, None, None, 0, 0, 1e-3, 1.0)]) == 0
    assert call([], n=-1) != 0 and b"negative count" in lib.gsb_last_error()
    assert call([good(6, 3)], N=-2, vis=256) != 0 and b"negative count" in lib.gsb_last_error()
    assert lib.gsb_adam_step(2, None, 0, None, 0.9, 0.999, 1e-8, None) != 0
    assert b"null table" in lib.gsb_last_error()
    assert call([T(16, None, 48, 64, 10, 0, 1e-3, 1.0)]) != 0 and b"null pointer" in lib.gsb_last_error()
    assert call([T(16, 32, 48, 66, 10, 0, 1e-3, 1.0)]) != 0 and b"misaligned" in lib.gsb_last_error()
    assert call([good(-1)]) != 0 and b"negative numel" in lib.gsb_last_error()
    # selective: every tensor has N * D elements, D >= 1; dense: N = 0
    assert call([good(30, 3), good(45, 3)], N=10, vis=256) != 0 and b"N * D" in lib.gsb_last_error()
    assert call([good(10, 0)], N=10, vis=256) != 0 and b"N * D" in lib.gsb_last_error()
    assert call([good(30)], N=10) != 0 and b"without a visibility" in lib.gsb_last_error()
    assert call([good(30)], b1=1.0) != 0 and b"betas" in lib.gsb_last_error()
    assert call([good(30)], b2=-0.1) != 0 and b"betas" in lib.gsb_last_error()
    assert call([good(30)], eps=float("nan")) != 0 and b"eps" in lib.gsb_last_error()


def test_adam_profile_id_sits_before_the_rgbd_pair():
    _, lib = _lib()
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    assert names[-3:] == ["adam", "draw_rgbd", "draw_backward_rgbd"]


def test_adam_kernel_is_sm90a_without_spills():
    L, _ = _lib()
    sass = subprocess.run(["cuobjdump", "-sass", L.LIB_PATH], capture_output=True, text=True).stdout
    assert set(re.findall(r"code for (sm_\w+)", sass)) == {"sm_90a"}
    funcs = re.split(r"\n\s*Function : ", sass)
    bodies = [f for f in funcs if re.match(r"\S*6k_adamILb[01]EE", f)]
    assert len(bodies) == 2  # the dense and the selective instantiation
    for body in bodies:
        assert "LDG.E.128" in body and "STG.E.128" in body  # the 16-byte path
    r = subprocess.run(["cuobjdump", "-res-usage", L.LIB_PATH], capture_output=True, text=True)
    found = re.findall(r"Function (\S*6k_adamILb[01]EE\S*):\s*\n\s*(REG:.*)", r.stdout)
    assert len(found) == 2
    for name, usage in found:
        assert "LOCAL:0 " in usage and "STACK:0 " in usage, (name, usage)
