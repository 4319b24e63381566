"""Density control and Gaussian record conversion at the sizes and values where their kernels
branch, against oracle/density_oracle.py:

- the plan (classify + the two-kernel scan + slots) on both sides of the classify CTA (1024 rows),
  of one scan warp (32 CTAs) and of k_density_scan_blocks' 1024-CTA span, whose carry only runs
  past 1 048 576 rows, with uniform, alternating and all-clone-CTA class layouts;
- the rebuild at the row-group edges (31-33, 255-257 rows) and at and past the row-group grid
  cap G = 8 * SMs * 256 rows, where warps loop over groups, with and without Adam moments, and the
  per-element kernel (N = 23 000 000) without them;
- every class threshold exactly at and one ulp on each side of its boundary;
- NaN / inf in every density input, and the clone / split arithmetic at its float32 edges;
- accumulate (first call, masks, an odd-offset dloss_dus view) and reset_alpha;
- PLY decode, get_training_params and save_training_params at every SH degree.

Index work (classes, slots, counts, moved rows, Adam moments) is bit-exact; recomputed values
agree to 3e-6 relative, non-finite values must match in kind and sign."""
import numpy as np
import pytest
import torch

from oracle import density_oracle as do

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAMES = do.NAMES
F = np.float32
KEEP, CLONE, SPLIT, PRUNE = do.KEEP, do.CLONE, do.SPLIT, do.PRUNE


def t(a, dtype=None):
    x = torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    return x.to(dtype) if dtype is not None else x


def n(x):
    return x.detach().cpu().numpy()


def close(got, want, name, rtol=3e-6, atol=2e-6):
    """finite values within rtol / atol; NaN and +-inf in the same places (and of the same sign)"""
    assert got.shape == want.shape, (name, got.shape, want.shape)
    fin = np.isfinite(want)
    assert np.array_equal(np.isfinite(got), fin), "%s: finite pattern differs" % name
    assert np.array_equal(got[~fin], want[~fin], equal_nan=True), "%s: non-finite values differ" % name
    err = np.abs(got[fin].astype(np.float64) - want[fin]) - (rtol * np.abs(want[fin]) + atol)
    assert (err <= 0).all(), "%s: max excess %.3e" % (name, err.max())


def ulp(x, k):
    """x moved k float32 ulps (k < 0: down)"""
    x = F(x)
    for _ in range(abs(k)):
        x = np.nextafter(x, F(np.inf) if k > 0 else F(-np.inf))
    return F(x)


def as_device_th(th_o):
    return {k: float(v) for k, v in th_o.items()}


def expected_slots(cls):
    flags = np.stack([cls != PRUNE, cls == CLONE, cls == SPLIT], axis=1).astype(np.int64)
    return np.cumsum(flags, axis=0) - flags, tuple(int(x) for x in flags.sum(axis=0))


def check_plan(alphas, scales, acc, cnt, th_o, want_cls=None):
    """density.plan on device tensors against do.classify and the prefix sums of its flags"""
    from easygaussiansplatting_b200 import density
    cls, slots, counts = density.plan(alphas, scales, acc, cnt, as_device_th(th_o))
    cls_o = do.classify(n(alphas), n(scales), n(acc), n(cnt), th_o)
    if want_cls is not None:
        assert np.array_equal(cls_o, want_cls)
    got = n(cls)
    bad = np.flatnonzero(got != cls_o)
    assert bad.size == 0, "classes differ at %d rows, first %s: got %s want %s" % (
        bad.size, bad[:8].tolist(), got[bad[:8]].tolist(), cls_o[bad[:8]].tolist())
    sl_o, counts_o = expected_slots(cls_o)
    sl = n(slots)
    bad = np.flatnonzero((sl != sl_o).any(axis=1))
    assert bad.size == 0, "slots differ from row %d (of %d rows)" % (bad[0], bad.size)
    assert counts == counts_o, (counts, counts_o)
    return cls, slots, counts


def plan_inputs(N, seed, sense=5.0, acc_scale=1.0):
    """random_state's class mix drawn on the device (host memory stays small at 5M rows)"""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    U = lambda shape, a, b: torch.empty(shape, device=DEV).uniform_(a, b, generator=gen)
    alphas = U((N, 1), -7.5, 4)
    scales = (U((N, 1), np.log(0.002 * sense), np.log(0.12 * sense)).exp_() * U((N, 3), 0.6, 1.5)).log_()
    cnt = torch.randint(0, 6, (N,), device=DEV, generator=gen, dtype=torch.int32)
    acc = torch.empty((N, 1), device=DEV).normal_(0.0, 1.5e-6 * acc_scale, generator=gen).abs_()
    return alphas, scales, acc.mul_((cnt > 0).unsqueeze(1)), cnt, gen


def full_state(N, seed, acc_scale=1.0, moments=True):
    alphas, scales, acc, cnt, gen = plan_inputs(N, seed, acc_scale=acc_scale)
    U = lambda shape, a, b: torch.empty(shape, device=DEV).uniform_(a, b, generator=gen)
    Nn = lambda shape, s=1.0: torch.empty(shape, device=DEV).normal_(0.0, s, generator=gen)
    P = dict(pws=U((N, 3), -2, 2), low_shs=Nn((N, 3)), high_shs=Nn((N, 45), 0.1), alphas_raw=alphas,
             scales_raw=scales, rots_raw=Nn((N, 4)).mul_(U((N, 1), 0.3, 2)))
    if not moments:
        return P, None, None, acc, cnt, gen
    M = {k: Nn(v.shape, 1e-3) for k, v in P.items()}
    V = {k: U(v.shape, 0.0, 1e-6) for k, v in P.items()}
    return P, M, V, acc, cnt, gen


# ------------------------------------------------------------------------------------------ plan

# 1023-1025: one classify CTA; 32 Ki (+1): one scan warp; 1 Mi - 1 .. 1 Mi + 1: nb = 1024 / 1025,
# the edge of k_density_scan_blocks' 1024-CTA span; 2 098 177: three span iterations; ~5M rows
@pytest.mark.parametrize("N", [1023, 1024, 1025, 32 * 1024, 32 * 1024 + 1, 1048575, 1048576, 1048577, 2098177,
                               5000011])
def test_plan_across_scan_spans(N):
    alphas, scales, acc, cnt, _ = plan_inputs(N, N % 9973)
    _, _, (K, Cn, S) = check_plan(alphas, scales, acc, cnt, do.thresholds(5.0))
    assert 0 < K < N and Cn > 0 and S > 0, (K, Cn, S)


# rows that take a given class with the sense-5 thresholds: (alphas_raw, scales_raw, acc, cnt)
CANON = {KEEP: (0.0, np.log(0.01), 0.0, 1), CLONE: (0.0, np.log(0.01), 1e-5, 1),
         SPLIT: (0.0, np.log(0.2), 1e-5, 1), PRUNE: (-10.0, np.log(0.01), 0.0, 1)}


def rows_of_classes(cls):
    tab = torch.tensor([CANON[c] for c in range(4)], dtype=torch.float64, device=DEV)[cls.long()]
    alphas = tab[:, 0:1].float().contiguous()
    scales = tab[:, 1:2].float().expand(-1, 3).contiguous()
    return alphas, scales, tab[:, 2:3].float().contiguous(), tab[:, 3].int().contiguous()


@pytest.mark.parametrize("N", [1048577, 2098177])
@pytest.mark.parametrize("layout", ["all_keep", "all_clone", "all_split", "all_prune", "alternating", "clone_ctas"])
def test_plan_class_layouts(N, layout):
    """uniform classes (a count of 1024 in one 16-bit half of the packed per-CTA count, or in
    both for all-clone), a class change every row, and random classes around whole CTAs of
    clones: 1023 / 1024 straddle the first span's end, 2048 starts the third span"""
    if layout.startswith("all_"):
        c = dict(all_keep=KEEP, all_clone=CLONE, all_split=SPLIT, all_prune=PRUNE)[layout]
        cls = torch.full((N,), c, dtype=torch.uint8, device=DEV)
    elif layout == "alternating":
        cls = (torch.arange(N, device=DEV) % 4).to(torch.uint8)
    else:
        gen = torch.Generator(device=DEV).manual_seed(N)
        cls = torch.randint(0, 4, (N,), device=DEV, generator=gen, dtype=torch.uint8)
        for b in (0, 1023, 1024, 2048):
            cls[b * 1024:(b + 1) * 1024] = CLONE
    _, _, counts = check_plan(*rows_of_classes(cls), do.thresholds(5.0), want_cls=n(cls))
    if layout == "all_prune":
        assert counts == (0, 0, 0)


# ----------------------------------------------------------------------------------------- apply

def row_count(spec):
    """N, or G = 8 * SMs * 256 (the row-group kernel's grid cap in rows) plus an offset"""
    if isinstance(spec, int):
        return spec
    G = 8 * torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count * 256
    return dict(G=G, G1=G + 1, G2=2 * G + 33)[spec]


def check_tail(dst, dP, cls, z, K):
    """the clone / split rows against do.densify run on only their source rows, in order: a new
    row depends on nothing but its source row and (splits) its row of z"""
    src = (cls == CLONE) | (cls == SPLIT)
    sub = {k: n(v[src]) for k, v in dP.items()}
    cls_sub = n(cls[src])
    oP, _, _, (Ks, Cs, Ss) = do.densify(sub, None, None, cls_sub, n(z))
    assert Ks == cls_sub.size and Ss == z.shape[0]
    for k in NAMES:
        close(n(dst[k][K:]), oP[k][Ks:], "tail " + k)
    for k in ("low_shs", "high_shs"):
        assert np.array_equal(n(dst[k][K:]), oP[k][Ks:]), k


@pytest.mark.parametrize("spec", [31, 32, 33, 255, 256, 257, "G", "G1", "G2"])
def test_apply_row_group_edges(spec):
    from easygaussiansplatting_b200 import density
    N = row_count(spec)
    P, M, V, acc, cnt, gen = full_state(N, 1000 + N % 7919)
    cls, slots, (K, Cn, S) = check_plan(P["alphas_raw"], P["scales_raw"], acc, cnt, do.thresholds(5.0))
    z = torch.empty((S, 3), device=DEV).normal_(0.0, 1.0, generator=gen)
    dst, dm, dv = density.apply(cls, slots, (K, Cn, S), P, M, V, z)
    dst0, dm0, dv0 = density.apply(cls, slots, (K, Cn, S), P, None, None, z)
    assert dm0 is None and dv0 is None
    for k in NAMES:
        assert torch.equal(dst0[k], dst[k]), k
    if N <= 300_000:
        hP, hM, hV = ({k: n(v) for k, v in X.items()} for X in (P, M, V))
        oP, oM, oV, ocounts = do.densify(hP, hM, hV, n(cls), n(z))
        assert ocounts == (K, Cn, S)
        for k in NAMES:
            assert np.array_equal(n(dst[k])[:K], oP[k][:K]), k
            close(n(dst[k]), oP[k], k)
            assert np.array_equal(n(dm[k]), oM[k]) and np.array_equal(n(dv[k]), oV[k]), k
        return
    keep = cls != PRUNE
    for k in NAMES:
        assert torch.equal(dst[k][:K], P[k][keep]), k
        assert torch.equal(dm[k][:K], M[k][keep]) and torch.equal(dv[k][:K], V[k][keep]), k
        assert not dm[k][K:].any() and not dv[k][K:].any(), k
    check_tail(dst, P, cls, z, K)


def test_apply_per_element_kernel_without_state():
    """N = 23 000 000, the smallest N the row-group kernel takes with 64-bit destination offsets,
    without Adam moments (six jobs).  Peak device memory: the parameters (236 B / row, 5.4 GB), the plan inputs and slots
    (25 B / row, 0.6 GB), the rebuilt parameters (<= 1.1 N rows, 6.0 GB) and one boolean gather
    of high_shs for the check (<= 4.1 GB): at most 16.1 GB, 13.9 GB with this seed on an H100."""
    from easygaussiansplatting_b200 import density
    N = 23_000_000
    need = 16 << 30
    free, total = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip("needs %d bytes of free device memory, %d of %d free" % (need, free, total))
    torch.cuda.reset_peak_memory_stats()
    P, _, _, acc, cnt, gen = full_state(N, 77, acc_scale=0.25, moments=False)   # few densified rows: a small host tail
    cls, slots, (K, Cn, S) = density.plan(P["alphas_raw"], P["scales_raw"], acc, cnt, density.raw_thresholds(5.0))
    assert K > 0 and Cn > 0 and S > 0 and K + Cn + S <= 1.1 * N, (K, Cn, S)
    z = torch.empty((S, 3), device=DEV).normal_(0.0, 1.0, generator=gen)
    dst, dm, dv = density.apply(cls, slots, (K, Cn, S), P, None, None, z)
    assert dm is None and dv is None
    keep = cls != PRUNE
    for k in NAMES:
        assert torch.equal(dst[k][:K], P[k][keep]), k
    check_tail(dst, P, cls, z, K)
    print("N %d: K %d C %d S %d, peak device memory %d bytes" % (N, K, Cn, S, torch.cuda.max_memory_allocated()))


# ------------------------------------------------------------------------------------ thresholds

def tie_rows(th_o):
    """(alphas_raw, scales_raw[3], acc, cnt) rows at and one ulp around every class boundary except
    the exp(s) clone bound, which needs the device's exp (test_threshold_ties)"""
    small, big_g = F(np.log(0.01)), F(1e-5)
    rows = []
    for a in (ulp(th_o["alpha_raw_min"], -1), th_o["alpha_raw_min"], ulp(th_o["alpha_raw_min"], 1)):
        rows += [(a, (small,) * 3, F(0), 1), (a, (small,) * 3, big_g, 1)]
    for col in range(3):
        for s in (ulp(th_o["scale_raw_max"], -1), th_o["scale_raw_max"], ulp(th_o["scale_raw_max"], 1)):
            sc = [small] * 3
            sc[col] = s
            rows += [(F(0), tuple(sc), F(0), 1), (F(0), tuple(sc), big_g, 1)]
    g = th_o["grad_min"]
    for acc in (ulp(g, -1), g, ulp(g, 1)):
        rows.append((F(0), (small,) * 3, acc, 1))
    # cnt = 3: every float32 accumulator near 3 g whose float32 quotient lands on, or next to, g
    three = [ulp(F(3) * g, k) for k in range(-6, 7)]
    q = np.array([F(a) / F(3) for a in three], F)
    assert (q == g).any() and (q < g).any() and (q > g).any(), "cnt 3 quotients do not straddle grad_min"
    rows += [(F(0), (small,) * 3, a, 3) for a in three]
    return rows


def tables(rows):
    alphas = np.array([[r[0]] for r in rows], F)
    scales = np.array([r[1] for r in rows], F)
    acc = np.array([[r[2]] for r in rows], F)
    cnt = np.array([r[3] for r in rows], np.int32)
    return alphas, scales, acc, cnt


@pytest.mark.parametrize("exact_clone_bound", [False, True])
def test_threshold_ties(exact_clone_bound):
    """alpha_raw_min (a < min prunes), scale_raw_max in each column (s > max prunes), grad_min
    (g >= min densifies) for cnt 1 and for a cnt-3 quotient that rounds onto it, and the clone
    bound max exp(s) <= scale_clone_max.  The exp rows are found with torch.exp on the device (the
    reference's arithmetic); exact_clone_bound moves the bound onto one of those exp values, so
    one row sits exactly on it"""
    th_o = do.thresholds(5.0)
    s0 = F(np.log(th_o["scale_clone_max"]))
    svals = np.array([ulp(s0, k) for k in range(-3, 4)], F)
    e_dev = n(torch.exp(t(svals)))
    if exact_clone_bound:
        th_o = dict(th_o, scale_clone_max=F(e_dev[3]))
    rows = tie_rows(th_o)
    first_exp = len(rows)
    small = F(np.log(0.01))
    for col in range(3):
        for s in svals:
            sc = [small] * 3
            sc[col] = s
            rows.append((F(0), tuple(sc), F(1e-5), 1))
    alphas, scales, acc, cnt = tables(rows)
    want = do.classify(alphas, scales, acc, cnt, th_o)
    dev_side = np.tile(np.where(e_dev <= th_o["scale_clone_max"], CLONE, SPLIT), 3)
    host_side = want[first_exp:]
    if not np.array_equal(host_side, dev_side):
        print("numpy exp puts %d clone-bound rows on the other side than torch.exp on the device; "
              "the device's answer is used for them" % int((host_side != dev_side).sum()))
    want[first_exp:] = dev_side
    assert (want == PRUNE).any() and (want == KEEP).any() and (want == CLONE).any() and (want == SPLIT).any()
    if exact_clone_bound:
        assert (e_dev == th_o["scale_clone_max"]).any()
    from easygaussiansplatting_b200 import density
    cls, slots, counts = density.plan(t(alphas), t(scales), t(acc), t(cnt), as_device_th(th_o))
    bad = np.flatnonzero(n(cls) != want)
    assert bad.size == 0, ["row %d %s: got %d want %d" % (i, rows[i], n(cls)[i], want[i]) for i in bad]
    sl_o, counts_o = expected_slots(want)
    assert np.array_equal(n(slots), sl_o) and counts == counts_o


# ------------------------------------------------------------------------------------ non-finite

NAN, INF = F(np.nan), F(np.inf)
SM, MID, BIG, GACC = F(np.log(0.01)), F(np.log(0.2)), F(1.0), F(1e-5)


def nonfinite_rows():
    """(label, alphas_raw, scales_raw[3], acc, cnt, zero quaternion, class the reference gives)"""
    R = [("alpha nan, densify", NAN, (SM,) * 3, GACC, 1, False, CLONE),
         ("alpha nan, keep", NAN, (SM,) * 3, F(0), 1, False, KEEP),
         ("alpha +inf clone", INF, (SM,) * 3, GACC, 1, False, CLONE),
         ("alpha -inf", -INF, (SM,) * 3, GACC, 1, False, PRUNE)]
    for col in range(3):
        sc = [SM] * 3
        sc[col] = NAN
        sc[(col + 1) % 3] = BIG
        R.append(("scale %d nan + big column, keep" % col, F(0), tuple(sc), F(0), 1, False, KEEP))
        R.append(("scale %d nan + big column, densify" % col, F(0), tuple(sc), GACC, 1, False, SPLIT))
        sc = [SM] * 3
        sc[col] = NAN
        R.append(("scale %d nan + small columns, densify" % col, F(0), tuple(sc), GACC, 1, False, SPLIT))
        sc = [SM] * 3
        sc[col] = INF
        R.append(("scale %d +inf" % col, F(0), tuple(sc), GACC, 1, False, PRUNE))
        sc = [SM] * 3
        sc[col] = -INF
        R.append(("scale %d -inf, clone" % col, F(0), tuple(sc), GACC, 1, False, CLONE))
    R += [("acc nan", F(0), (SM,) * 3, NAN, 1, False, KEEP),
          ("acc +inf", F(0), (SM,) * 3, INF, 1, False, CLONE),
          ("acc +inf, cnt 2", F(0), (MID,) * 3, INF, 2, False, SPLIT),
          ("cnt 0, acc 0", F(0), (SM,) * 3, F(0), 0, False, KEEP),
          ("cnt 0, acc > 0, clone", F(0), (SM,) * 3, F(1e-9), 0, False, CLONE),
          ("cnt 0, acc > 0, split", F(0), (MID,) * 3, F(1e-9), 0, False, SPLIT),
          ("zero quaternion clone", F(1), (SM,) * 3, GACC, 1, True, CLONE),
          ("zero quaternion split", F(1), (MID, SM, SM), GACC, 1, True, SPLIT)]
    for a in (17.33, 17.5, 30.0, 88.0):
        R.append(("alpha %g clone" % a, F(a), (SM,) * 3, GACC, 1, False, CLONE))
    for a in (9.5, 12.0, 16.0):
        R.append(("alpha %g split" % a, F(a), (MID, SM, SM), GACC, 1, False, SPLIT))
    for s in (-87.5, -90.0, -100.0, -103.0, -103.5, -104.0, -110.0):
        R.append(("split scale %g" % s, F(0.5), (MID, F(s), F(s)), GACC, 1, False, SPLIT))
        R.append(("clone scale %g" % s, F(0.5), (F(s), SM, F(s)), GACC, 1, False, CLONE))
    return R


def test_nonfinite_inputs():
    """NaN and +-inf in alphas_raw, each scale column and the accumulators, cnt = 0, zero
    quaternions, saturated sigmoids and scales whose exp underflows, through plan and apply.  A
    NaN scale is neither pruned for size nor cloned (torch.max propagates NaN): with a gradient it
    splits, and the split rows are NaN (the reference's torch.normal raises on a NaN std)."""
    from easygaussiansplatting_b200 import density
    R = nonfinite_rows()
    m = len(R)
    rng = np.random.default_rng(4)
    alphas, scales, acc, cnt = tables([(r[1], r[2], r[3], r[4]) for r in R])
    want = np.array([r[6] for r in R], np.uint8)
    P = dict(pws=rng.uniform(-2, 2, (m, 3)), low_shs=rng.normal(size=(m, 3)), high_shs=rng.normal(size=(m, 45)),
             alphas_raw=alphas, scales_raw=scales, rots_raw=rng.normal(size=(m, 4)))
    P = {k: v.astype(F) for k, v in P.items()}
    P["rots_raw"][[r[5] for r in R]] = 0
    M = {k: (rng.normal(size=v.shape) * 1e-3).astype(F) for k, v in P.items()}
    V = {k: rng.uniform(size=v.shape).astype(F) for k, v in P.items()}
    dP, dM, dV = ({k: t(v) for k, v in X.items()} for X in (P, M, V))
    cls, slots, (K, Cn, S) = density.plan(dP["alphas_raw"], dP["scales_raw"], t(acc), t(cnt),
                                          density.raw_thresholds(5.0))
    got = n(cls)
    cls_o = do.classify(alphas, scales, acc, cnt, do.thresholds(5.0))
    assert np.array_equal(cls_o, want), [R[i][0] for i in np.flatnonzero(cls_o != want)]
    assert np.array_equal(got, want), ["%s: %d, want %d" % (R[i][0], got[i], want[i])
                                      for i in np.flatnonzero(got != want)]
    sl_o, counts_o = expected_slots(want)
    assert np.array_equal(n(slots), sl_o) and (K, Cn, S) == counts_o
    z = rng.normal(size=(S, 3)).astype(F)
    dst, dm, dv = density.apply(cls, slots, (K, Cn, S), dP, dM, dV, t(z))
    with np.errstate(all="ignore"):
        oP, oM, oV, _ = do.densify(P, M, V, want, z)
    # logit(sigmoid(x)) loses most of its bits for |x| > 9 (1 - sigmoid(x) keeps a few): those
    # new rows are compared with torch's CUDA sigmoid / log instead of numpy's
    src = np.concatenate([np.flatnonzero(want == CLONE), np.flatnonzero(want == SPLIT)])
    ill = np.abs(alphas[src, 0]) > 9
    new_a = n(dst["alphas_raw"])[K:]
    sig = torch.sigmoid(t(alphas[src[ill]]))
    ref_ill = n(torch.log(sig / (1 - sig)))
    close(new_a[ill], ref_ill, "alphas_raw, |x| > 9 vs torch CUDA")
    print("new alphas_raw for |alphas_raw| > 9 (%d rows): %s torch's CUDA sigmoid / log bit for bit" % (
        int(ill.sum()), "equal to" if np.array_equal(new_a[ill], ref_ill, equal_nan=True) else "NOT equal to"))
    oP["alphas_raw"][K:][ill] = new_a[ill]
    for k in NAMES:
        assert np.array_equal(n(dst[k])[:K], oP[k][:K], equal_nan=True), k
        close(n(dst[k]), oP[k], k)
        assert np.array_equal(n(dm[k]), oM[k]) and np.array_equal(n(dv[k]), oV[k]), k
    # the split rows of a NaN scale are NaN, as is the new alpha of a NaN alpha
    nan_split = [i for i, r in enumerate(R) if r[6] == SPLIT and np.isnan(r[2]).any()]
    pos = {int(s): K + j for j, s in enumerate(src)}
    assert all(np.isnan(n(dst["pws"][pos[i]])).all() for i in nan_split)


# ---------------------------------------------------------------------------- accumulate / reset

@pytest.mark.parametrize("N", [1, 257, 1048577])
@pytest.mark.parametrize("kind", ["none", "all", "random"])
def test_accumulate_vs_oracle(N, kind):
    """five update_density_info steps; the first stores every row's norm (masked-out rows too)
    and counts the mask.  An odd-offset dloss_dus view (scalar loads) must agree bit for bit."""
    from easygaussiansplatting_b200 import density
    gen = torch.Generator(device=DEV).manual_seed(N + len(kind))
    acc = torch.empty((N, 1), device=DEV)
    cnt = torch.empty(N, dtype=torch.int32, device=DEV)
    acc2, cnt2 = torch.empty_like(acc), torch.empty_like(cnt)
    buf = torch.empty(2 * N + 1, device=DEV)
    acc_o = cnt_o = None
    for step in range(5):
        dus = torch.empty((N, 2), device=DEV).normal_(0.0, 1e-6, generator=gen)
        if kind == "random":
            mask = torch.rand(N, device=DEV, generator=gen) < 0.5
        else:
            mask = torch.full((N,), kind == "all", dtype=torch.bool, device=DEV)
        density.accumulate(dus, mask, acc, cnt, step == 0)
        odd = buf[1:].view(N, 2)
        assert odd.data_ptr() % 8 == 4
        odd.copy_(dus)
        density.accumulate(odd, mask, acc2, cnt2, step == 0)
        acc_o, cnt_o = do.accumulate(n(dus), n(mask), acc_o, cnt_o)
        assert np.array_equal(n(cnt), cnt_o), step
        close(n(acc), acc_o, "grad_accum step %d" % step, rtol=1e-6, atol=0)
        assert torch.equal(acc2, acc) and torch.equal(cnt2, cnt), step


@pytest.mark.parametrize("state", [True, False])
def test_reset_alpha_vs_oracle(state):
    """clamp from above at logit(0.01), bit for bit, including rows on the reset value, one ulp
    around it, +-inf and NaN (NaN > v is false: kept); with moments they are zeroed, without
    them the optimizer state stays empty"""
    from easygaussiansplatting_b200.density import DensityController
    from easygaussiansplatting_b200.gau_io import adam_groups
    N = 100_003
    rng = np.random.default_rng(11)
    v = F(np.log(0.01 / (1 - 0.01)))
    a = rng.uniform(-8, 8, (N, 1)).astype(F)
    a[:7, 0] = [v, ulp(v, -1), ulp(v, 1), np.nan, np.inf, -np.inf, F(0)]
    params = {k: torch.zeros((N, w), device=DEV).requires_grad_() for k, w in zip(NAMES, (3, 3, 45, 1, 3, 4))}
    params["alphas_raw"] = t(a).requires_grad_()
    opt = torch.optim.Adam(adam_groups(params), lr=0.0, eps=1e-15)
    if state:
        for g in opt.param_groups:
            p = g["params"][0]
            opt.state[p] = {"step": torch.tensor(1.0), "exp_avg": torch.ones_like(p), "exp_avg_sq": torch.ones_like(p)}
    DensityController(5.0, verbose=False).reset_alpha(params, opt)
    want, zm, zv = do.reset_alpha(a)
    assert np.array_equal(n(params["alphas_raw"]), want, equal_nan=True)
    pa = params["alphas_raw"]
    if state:
        assert np.array_equal(n(opt.state[pa]["exp_avg"]), zm) and np.array_equal(n(opt.state[pa]["exp_avg_sq"]), zv)
        assert all(bool((opt.state[g["params"][0]]["exp_avg"] == 1).all()) for g in opt.param_groups
                   if g["name"] != "alphas_raw")
    else:
        assert len(opt.state) == 0


# -------------------------------------------------------------------------------- record conversion

def ply_names(sh_dim):
    return (["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] +
            ["f_rest_%d" % i for i in range(sh_dim - 3)] +
            ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"])


def write_ply(path, N, sh_dim, seed, shuffled):
    rng = np.random.default_rng(seed)
    names = ply_names(sh_dim)
    cols = {nm: rng.normal(size=N).astype(F) for nm in names}
    cols["opacity"] = rng.uniform(-12, 12, N).astype(F)
    for i in range(3):
        cols["scale_%d" % i] = rng.uniform(-7, 1, N).astype(F)
    for nm in ("nx", "ny", "nz"):
        cols[nm][:] = 0
    if shuffled:
        names = [names[i] for i in rng.permutation(len(names))]
    head = "ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % N
    head += "".join("property float %s\n" % nm for nm in names) + "end_header\n"
    raw = head.encode("ascii") + np.stack([cols[nm] for nm in names], axis=1).astype("<f4").tobytes()
    with open(path, "wb") as f:
        f.write(raw)
    return raw


@pytest.mark.parametrize("sh_dim", [3, 12, 27, 48])
@pytest.mark.parametrize("N", [1, 7, 40000])
@pytest.mark.parametrize("shuffled", [False, True])
def test_record_conversion_every_sh_degree(sh_dim, N, shuffled, tmp_path):
    """load_ply (f_rest transpose for k = 0, 3, 8, 15 coefficients per channel), get_training_params
    (0.001 padding of high_shs from column sh_dim - 3; alpha 0 / 1 -> -inf / +inf, scale 0 -> -inf)
    and save_training_params' arithmetic, against the oracle.  40 000 rows x 59 columns is past
    the stream grid's cap, so every kernel grid-strides."""
    from easygaussiansplatting_b200 import gau_io
    p = str(tmp_path / "scene.ply")
    raw = write_ply(p, N, sh_dim, 100 * sh_dim + N, shuffled)
    gs = gau_io.load_ply(p)
    want = do.decode_ply(raw)
    assert gs.dtype == want.dtype
    for k in ("pw", "sh"):
        assert np.array_equal(np.asarray(gs[k]), np.asarray(want[k])), k
    for k in ("rot", "scale", "alpha"):
        close(np.asarray(gs[k]), np.asarray(want[k]), k, rtol=2e-6, atol=1e-7)

    edge = want.copy()
    edge["alpha"][0] = 0
    edge["scale"][0, 1] = 0
    if N > 1:
        edge["alpha"][1] = 1
        edge["scale"][1] = 0
    params, _ = gau_io.get_training_params(edge)
    with np.errstate(divide="ignore"):
        tp = do.training_params(edge)
    for k in ("pws", "low_shs", "high_shs", "rots_raw"):
        assert np.array_equal(n(params[k]), tp[k]), k
    assert (n(params["high_shs"])[:, sh_dim - 3:] == F(0.001)).all()
    for k in ("alphas_raw", "scales_raw"):
        close(n(params[k]), tp[k], "training " + k)
    assert n(params["alphas_raw"])[0, 0] == -np.inf and n(params["scales_raw"])[0, 1] == -np.inf
    if N > 1:
        assert n(params["alphas_raw"])[1, 0] == np.inf

    rows = gau_io.params_to_gs_rows(params)
    back = do.params_to_gs({k: n(v) for k, v in params.items()})
    flat = np.ascontiguousarray(back).view("<f4").reshape(N, 59)
    close(n(rows), flat, "params_to_gs", rtol=3e-6, atol=1e-7)
