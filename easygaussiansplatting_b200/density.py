"""Density control on the C ABI (SURVEY 8f row N3): the mirror of the density half of
gsplat.gsmodel.GSModel (reference gsplat/gsmodel.py:168-331) and of prune_params /
update_params (:132-166).

    ctl = DensityController(sense_size)
    ctl.update_density_info(us.grad, mask)            # every iteration, after backward
    ctl.update_gaussian_density(params, optimizer)    # every few epochs
    ctl.reset_alpha(params, optimizer)

`params` is the reference's dict of six leaf tensors, `optimizer` a torch.optim.Adam whose
param groups carry the reference's "name" keys (get_training_params, gsmodel.py:114-127).
The parameters and both Adam moments are rebuilt by ONE kernel pass (gsb_density_apply)
instead of 18 boolean-index + torch.cat round trips.  Split offsets use unit normals drawn
with the SAME torch generator call sequence as the reference (torch.normal(mean, std) is
normal_(0, 1) * std + mean), so a run seeded like the reference splits identically.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import GAUSSIAN_TENSORS, GAUSSIAN_WIDTHS, Gaussians


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _check(t, name, shape=None, dtype=torch.float32):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise ValueError("%s must be a CUDA tensor (there is no CPU fallback)" % name)
    if t.dtype != dtype:
        raise ValueError("%s must be %s, got %s" % (name, dtype, t.dtype))
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise ValueError("%s must have shape %s, got %s" % (name, tuple(shape), tuple(t.shape)))
    return t.contiguous()


def gaussians_struct(tensors):
    """dict of the six tensors -> (gsb_gaussians, keep-alive list)"""
    g, keep = Gaussians(), []
    for k in GAUSSIAN_TENSORS:
        t = tensors[k]
        keep.append(t)
        setattr(g, k, t.data_ptr())
    return g, keep


def _structs(*dicts):
    """-> (C.byref gsb_gaussians of each dict of the six tensors, None for None; keep-alive list)"""
    structs, keep = [], []
    for d in dicts:
        if d is None:
            structs.append(None)
        else:
            g, ka = gaussians_struct(d)
            keep.append((g, ka))
            structs.append(C.byref(g))
    return structs, keep


def _copy(t, name, shape):
    """a checked contiguous float32 CUDA view of `shape` (a copy if `t` is not contiguous)"""
    return _check(t.detach(), name, shape)


def _in_place(t, name, shape):
    """the tensor itself (contiguous float32 CUDA of `shape`): the kernels write through its pointer"""
    c = _check(t.detach(), name, shape)
    if c.data_ptr() != t.data_ptr():
        raise ValueError("%s must be contiguous (it is updated in place)" % name)
    return c


def gather_state(params, optimizer, extra, take):
    """checked (N, tensors, Adam moments m / v or None, groups) of the six tensors and the [N, D]
    `extra` entries of `params`; take: _copy or _in_place.  The moments are those of the optimizer
    groups named after the tensors, for all of them or for none."""
    N = params["pws"].shape[0]
    src = {}
    for k, w in zip(GAUSSIAN_TENSORS, GAUSSIAN_WIDTHS):
        src[k] = take(params[k], "params[%r]" % k, (N, w))
    for k in extra:
        if k in GAUSSIAN_TENSORS:
            raise ValueError("extra names a built-in tensor: %r" % (k,))
        t = params[k]
        if not (isinstance(t, torch.Tensor) and t.dim() == 2 and t.shape[0] == N and t.shape[1] >= 1):
            raise ValueError("params[%r] must be [N, D] with N = %d and D >= 1" % (k, N))
        src[k] = take(t, "params[%r]" % (k,), tuple(t.shape))
    groups = {g["name"]: g for g in optimizer.param_groups}
    names = GAUSSIAN_TENSORS + tuple(extra)
    missing = [k for k in names if k not in groups]
    if missing:
        raise ValueError("the optimizer has no param group named %s" % ", ".join(map(repr, missing)))
    states = {k: optimizer.state.get(groups[k]["params"][0], None) for k in names}
    have = [s is not None and "exp_avg" in s for s in states.values()]
    if any(have) and not all(have):
        raise ValueError("optimizer state must exist for all groups or for none")
    m = v = None
    if all(have):
        m = {k: take(states[k]["exp_avg"], "exp_avg[%r]" % k, src[k].shape) for k in names}
        v = {k: take(states[k]["exp_avg_sq"], "exp_avg_sq[%r]" % k, src[k].shape) for k in names}
    return N, src, m, v, groups


def swap_parameters(params, optimizer, groups, dst, dst_m, dst_v):
    """params[k] and the optimizer group k become a new Parameter of dst[k] for every k in dst; the
    group's optimizer state moves to it with the moments dst_m[k] / dst_v[k] (none without them)"""
    for k in dst:
        group = groups[k]
        old = group["params"][0]
        new = torch.nn.Parameter(dst[k].requires_grad_(True))
        st = optimizer.state.pop(old, None)
        if st is not None and dst_m is not None:
            st["exp_avg"], st["exp_avg_sq"] = dst_m[k], dst_v[k]
            optimizer.state[new] = st
        group["params"][0] = new
        params[k] = new


def report(verbose, title, rows):
    """the reference's printed report: "gaussian <title> report", then "<name>:  <value>" rows"""
    if verbose:
        print("---------------------")
        print("gaussian %s report" % title)
        for name, val in rows:
            print("%s: " % name, val)
        print("---------------------")


def raw_thresholds(sense_size, alpha_threshold=0.005, grad_threshold=4e-7):
    """GSModel.__init__ (gsmodel.py:170-181) in the units the kernels compare in"""
    f = np.float32
    return dict(alpha_raw_min=float(f(np.log(alpha_threshold / (1 - alpha_threshold)))),
                scale_raw_max=float(f(np.log(0.1 * sense_size))), grad_min=float(f(grad_threshold)),
                scale_clone_max=float(f(0.01 * sense_size)))


def accumulate(dloss_dus, mask, grad_accum, cunt, first):
    """gsb_density_accumulate on caller-owned accumulators"""
    lib = _lib.load()
    N = dloss_dus.shape[0]
    dus = _check(dloss_dus.detach().reshape(N, 2), "dloss_dus", (N, 2))
    m = _check(mask, "mask", (N,), torch.bool)
    _lib.check(lib.gsb_density_accumulate(N, _ptr(dus), _ptr(m), _ptr(grad_accum), _ptr(cunt), int(first), _stream()), lib)


def plan(alphas_raw, scales_raw, grad_accum, cunt, th):
    """-> (cls uint8 [N], slots int32 [N,3], (K, C, S)).  Waits for the counts (one D2H)."""
    lib = _lib.load()
    N = alphas_raw.shape[0]
    dev = alphas_raw.device
    cls = torch.empty(N, dtype=torch.uint8, device=dev)
    slots = torch.empty((N, 3), dtype=torch.int32, device=dev)
    nbytes = lib.gsb_density_workspace_bytes(N)
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    counts = (C.c_int64 * 3)()
    _lib.check(lib.gsb_density_plan(N, _ptr(alphas_raw), _ptr(scales_raw), _ptr(grad_accum), _ptr(cunt),
                                    th["alpha_raw_min"], th["scale_raw_max"], th["grad_min"], th["scale_clone_max"],
                                    _ptr(ws), nbytes, _ptr(cls), _ptr(slots), counts, _stream()), lib)
    return cls, slots, (int(counts[0]), int(counts[1]), int(counts[2]))


def apply(cls, slots, counts, src, src_m, src_v, z):
    """gsb_density_apply -> (dst, dst_m, dst_v) dicts of fresh tensors with K + C + S rows"""
    lib = _lib.load()
    K, Cn, S = counts
    N = cls.shape[0]
    dev = cls.device
    rows = K + Cn + S

    def fresh():
        return {k: torch.empty((rows, w), dtype=torch.float32, device=dev)
                for k, w in zip(GAUSSIAN_TENSORS, GAUSSIAN_WIDTHS)}

    dst = fresh()
    state = src_m is not None
    dst_m, dst_v = (fresh(), fresh()) if state else (None, None)
    structs, keep = _structs(src, src_m, src_v, dst, dst_m, dst_v)
    _lib.check(lib.gsb_density_apply(N, _ptr(cls), _ptr(slots), K, Cn, S, structs[0], structs[1], structs[2], _ptr(z),
                                     structs[3], structs[4], structs[5], _stream()), lib)
    return dst, dst_m, dst_v


def apply_rows(cls, slots, counts, src, src_m=None, src_v=None):
    """gsb_density_apply_rows on one [N, D] tensor (and its Adam moments, both or neither)
    -> (dst, dst_m, dst_v) fresh [K + C + S, D] tensors (the moments None without them)"""
    lib = _lib.load()
    K, Cn, S = counts
    N, D = src.shape
    dev = cls.device
    fresh = lambda: torch.empty((K + Cn + S, D), dtype=torch.float32, device=dev)  # noqa: E731
    dst = fresh()
    dst_m, dst_v = (fresh(), fresh()) if src_m is not None else (None, None)
    _lib.check(lib.gsb_density_apply_rows(N, _ptr(cls), _ptr(slots), K, Cn, S, D, _ptr(src), _ptr(src_m), _ptr(src_v),
                                          _ptr(dst), _ptr(dst_m), _ptr(dst_v), _stream()), lib)
    return dst, dst_m, dst_v


def plan_keep(keep):
    """gsb_density_plan_keep -> (cls uint8 [N], slots int32 [N,3], (K, 0, 0)).  Waits for K (one D2H)."""
    lib = _lib.load()
    N = keep.shape[0]
    dev = keep.device
    cls = torch.empty(N, dtype=torch.uint8, device=dev)
    slots = torch.empty((N, 3), dtype=torch.int32, device=dev)
    nbytes = lib.gsb_density_workspace_bytes(N)
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    counts = (C.c_int64 * 3)()
    _lib.check(lib.gsb_density_plan_keep(N, _ptr(keep), _ptr(ws), nbytes, _ptr(cls), _ptr(slots), counts, _stream()),
               lib)
    return cls, slots, (int(counts[0]), int(counts[1]), int(counts[2]))


@torch.no_grad()
def prune(params, optimizer, keep, extra=(), verbose=True):
    """Removes the Gaussians where keep[N] (bool, CUDA) is False: the six tensors of `params`, the
    [N, D] `extra` entries (per-Gaussian features) and their Adam moments, through one plan scan
    (gsb_density_plan_keep) and the density rebuild (gsb_density_apply / _rows).  Survivors keep
    their order and their moments; the optimizer groups get the new Parameters, and the other
    fields of their state (`step`) are left as they were.  Works with torch.optim.Adam and
    GaussianAdam, with or without optimizer state.  Prints the reference-style report when verbose.
    A captured GraphedFusedStep must be captured again afterwards.  -> dict(pruned, total)"""
    extra = tuple(extra)
    N, src, src_m, src_v, groups = gather_state(params, optimizer, extra, _copy)
    keep = _check(keep, "keep", (N,), torch.bool)
    if keep.device != src["pws"].device:
        raise ValueError("keep must be on the device of the parameters")
    cls, slots, counts = plan_keep(keep)
    K = counts[0]
    dst, dst_m, dst_v = apply(cls, slots, counts, src, src_m, src_v, None)
    for k in extra:
        dst[k], dm, dv = apply_rows(cls, slots, counts, src[k], src_m[k] if src_m else None, src_v[k] if src_v else None)
        if dst_m is not None:
            dst_m[k], dst_v[k] = dm, dv
    swap_parameters(params, optimizer, groups, dst, dst_m, dst_v)
    report(verbose, "prune", [("pruned num", N - K), ("total gaussian number", K)])
    return dict(pruned=N - K, total=K)


def lowest(score, fraction):
    """A keep mask over score[N] that drops exactly floor(fraction * N) rows: those with the lowest
    scores, ties broken by the lower index (a stable ascending sort), so the mask is deterministic.
    -> bool [N] on the device of score"""
    if not isinstance(score, torch.Tensor) or score.dim() != 1:
        raise ValueError("score must be a 1-D tensor")
    if not 0.0 <= float(fraction) <= 1.0:
        raise ValueError("fraction must be in [0, 1]")
    N = score.shape[0]
    n_drop = int(np.floor(float(fraction) * N))
    keep = torch.ones(N, dtype=torch.bool, device=score.device)
    order = torch.sort(score, stable=True).indices
    keep[order[:n_drop]] = False
    return keep


class DensityController:
    """the density-control half of gsplat.gsmodel.GSModel (gsmodel.py:168-331), same attribute
    names (`grad_accum`, `cunt`) and the same printed report.

    grad_threshold: the mean per-view |statistic| at or above which a Gaussian is cloned or split
    (the reference's 4e-7 by default).  Absolute-gradient densification (AbsGS) feeds
    update_density_info the `us_abs.grad` of the fused classes instead of `us.grad`; each view's
    norm is then >= the signed one, so the default threshold densifies more.  gsplat raises its
    threshold 4x for absgrad; no threshold for the absolute statistic has been measured with this
    library, so tune it for the scene."""

    def __init__(self, sense_size, verbose=True, grad_threshold=4e-7):
        self.grad_threshold = grad_threshold
        self.scale_threshold = 0.01 * sense_size
        self.alpha_threshold = 0.005
        self.big_threshold = 0.1 * sense_size
        self.reset_alpha_val = 0.01
        self.th = raw_thresholds(sense_size, self.alpha_threshold, self.grad_threshold)
        self.grad_accum = None
        self.cunt = None
        self.verbose = verbose

    def update_density_info(self, dloss_dus, mask):
        """gsmodel.py:219-234 (the caller passes us.grad -- or, for absolute-gradient
        densification, us_abs.grad of the fused classes -- and the GSFunction mask)"""
        N = dloss_dus.shape[0]
        first = self.cunt is None
        if first:
            self.grad_accum = torch.empty((N, 1), dtype=torch.float32, device=dloss_dus.device)
            self.cunt = torch.empty(N, dtype=torch.int32, device=dloss_dus.device)
        accumulate(dloss_dus, mask, self.grad_accum, self.cunt, first)

    @torch.no_grad()
    def update_gaussian_density(self, params, optimizer, generator=None, extra=()):
        """gsmodel.py:236-318 with prune_params / update_params (:132-166) fused in.  Mutates
        `params` and the optimizer's groups / state like the reference; returns the report.
        extra: names of further per-Gaussian [N, D] entries of `params` (per-Gaussian features),
        each with an optimizer group of that name; they are rebuilt by the same plan (survivors in
        order, then clones, then splits, every new row a copy of its source row, with zero Adam
        moments) by gsb_density_apply_rows.  extra=() is exactly the six-tensor update."""
        if self.cunt is None:
            raise RuntimeError("update_gaussian_density needs at least one update_density_info call")
        extra = tuple(extra)
        N, src, src_m, src_v, groups = gather_state(params, optimizer, extra, _copy)
        cls, slots, (K, Cn, S) = plan(src["alphas_raw"], src["scales_raw"], self.grad_accum, self.cunt, self.th)
        # the reference's torch.normal(mean=zeros(S,3), std=scales[split]) (:276-277)
        z = torch.empty((S, 3), dtype=torch.float32, device=src["pws"].device).normal_(0, 1, generator=generator)
        dst, dst_m, dst_v = apply(cls, slots, (K, Cn, S), src, src_m, src_v, z)
        for k in extra:
            dst[k], dm, dv = apply_rows(cls, slots, (K, Cn, S), src[k], src_m[k] if src_m else None,
                                        src_v[k] if src_v else None)
            if dst_m is not None:
                dst_m[k], dst_v[k] = dm, dv
        swap_parameters(params, optimizer, groups, dst, dst_m, dst_v)
        report(self.verbose, "density update", [("pruned num", N - K), ("cloned num", Cn), ("splited num", S),
                                                ("total gaussian number", K + Cn + S)])
        self.grad_accum = None
        self.cunt = None
        return dict(pruned=N - K, cloned=Cn, splited=S, total=K + Cn + S)

    def prune(self, params, optimizer, keep, extra=()):
        """`prune` with this controller's verbosity.  It also drops the accumulated densification
        statistics (`grad_accum`, `cunt`): they are indexed by the old rows, so the next
        update_gaussian_density needs update_density_info calls made after the prune."""
        out = prune(params, optimizer, keep, extra, self.verbose)
        self.grad_accum = None
        self.cunt = None
        return out

    @torch.no_grad()
    def reset_alpha(self, params, optimizer):
        """gsmodel.py:320-331"""
        lib = _lib.load()
        val = float(np.float32(np.log(self.reset_alpha_val / (1 - self.reset_alpha_val))))
        p = params["alphas_raw"]
        a = _check(p.detach(), "params['alphas_raw']")
        if a.data_ptr() != p.data_ptr():
            raise ValueError("params['alphas_raw'] must be contiguous")
        group = [g for g in optimizer.param_groups if g["name"] == "alphas_raw"][0]
        st = optimizer.state.get(group["params"][0], None)
        m = v = None
        if st is not None and "exp_avg" in st:
            m, v = _check(st["exp_avg"], "exp_avg"), _check(st["exp_avg_sq"], "exp_avg_sq")
        _lib.check(lib.gsb_reset_alpha(a.shape[0], _ptr(a), _ptr(m), _ptr(v), val, _stream()), lib)


# ----------------------------------------------------------------------------- MCMC densification

MCMC_RELOCATE, MCMC_GROW = 0, 1


def mcmc_plan(alphas_raw, alpha_raw_min, mode, n_draws):
    """gsb_mcmc_plan -> (workspace for up to n_draws draws, W_total, dead count).  Waits for the
    two counts (one D2H)."""
    lib = _lib.load()
    N = alphas_raw.shape[0]
    nbytes = lib.gsb_mcmc_workspace_bytes(N, n_draws)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=alphas_raw.device)
    counts = (C.c_int64 * 2)()
    _lib.check(lib.gsb_mcmc_plan(N, _ptr(alphas_raw), float(alpha_raw_min), mode, _ptr(ws), nbytes, counts,
                                 _stream()), lib)
    return ws, int(counts[0]), int(counts[1])


def mcmc_sample(ws, N, u):
    """gsb_mcmc_sample: fp64 uniforms u[n] -> int32 row ids [n] (after mcmc_plan on ws)"""
    lib = _lib.load()
    u = _check(u, "u", (u.shape[0],), torch.float64)
    sampled = torch.empty(u.shape[0], dtype=torch.int32, device=u.device)
    _lib.check(lib.gsb_mcmc_sample(N, u.shape[0], _ptr(u), _ptr(ws), ws.numel(), _ptr(sampled), _stream()), lib)
    return sampled


class MCMCController:
    """MCMC densification (Kheradmand et al., "3D Gaussian Splatting as Markov Chain Monte Carlo",
    2024; gsplat's MCMCStrategy): at most `cap_max` Gaussians, dead ones (opacity <= min_opacity)
    moved onto live ones instead of pruned, and covariance-shaped position noise every step.

        ctl = MCMCController(cap_max=1_000_000)
        optimizer.step(); ctl.inject_noise(params, optimizer)     # every step
        ctl.relocate(params, optimizer); ctl.grow(params, optimizer)  # every refinement interval

    `params` / `optimizer` are those of DensityController (six raw tensors, Adam groups named after
    them).  Sources are drawn in proportion to their opacity with an integer sampler whose ids do not
    depend on the GPU's summation order; the uniforms and normals come from `generator` (a CUDA
    torch.Generator, or the default one), so ranks that seed it alike stay identical.  A source hit
    c times shares its opacity among r = min(c + 1, n_max) copies with a scale that keeps the
    rendered footprint (DESIGN 3.11); the Adam moments of every row a call writes are zeroed."""

    NOISE_K, NOISE_X0 = 100.0, 0.995

    def __init__(self, cap_max, min_opacity=0.005, n_max=51, grow_rate=0.05, noise_lr=5e5, verbose=True):
        if not 1 <= int(n_max) <= 51:
            raise ValueError("n_max must be in [1, 51]")
        if not 0.0 < min_opacity < 1.0:
            raise ValueError("min_opacity must be in (0, 1)")
        self.cap_max = int(cap_max)
        self.min_opacity = float(min_opacity)
        self.n_max = int(n_max)
        self.grow_rate = float(grow_rate)
        self.noise_lr = float(noise_lr)
        self.verbose = verbose
        # the fp32 logit the kernels compare alphas_raw with, as raw_thresholds computes it
        self.alpha_raw_min = float(np.float32(np.log(self.min_opacity / (1 - self.min_opacity))))

    @torch.no_grad()
    def relocate(self, params, optimizer, generator=None, extra=()):
        """Moves every dead Gaussian (!(alphas_raw > logit(min_opacity)), NaN included) onto a live
        one drawn by opacity, in place: N and the Parameter objects stay.  The sources get their
        relocation value, dead row dead[j] (ascending) becomes a copy of the updated source j, and the
        Adam moments of sources and destinations are zeroed.  extra: names of further [N, D]
        entries of `params` with optimizer groups of those names (copied along).  HOST
        SYNCHRONISATION: one read of the dead count.  -> dict(relocated, total)"""
        lib = _lib.load()
        extra = tuple(extra)
        N, src, m, v, _ = gather_state(params, optimizer, extra, _in_place)
        n = 0
        if N:
            ws, w_total, n = mcmc_plan(src["alphas_raw"], self.alpha_raw_min, MCMC_RELOCATE, N)
            if w_total == 0:
                n = 0  # nothing alive to copy from
        if n:
            u = torch.rand(n, dtype=torch.float64, device=src["pws"].device, generator=generator)
            sampled = mcmc_sample(ws, N, u)
            structs, keep = _structs(src, m, v)
            _lib.check(lib.gsb_mcmc_relocate(N, n, _ptr(sampled), _ptr(ws), ws.numel(), self.min_opacity, self.n_max,
                                             *structs, _stream()), lib)
            for k in extra:
                _lib.check(lib.gsb_mcmc_relocate_rows(N, n, _ptr(sampled), _ptr(ws), ws.numel(), src[k].shape[1],
                                                      _ptr(src[k]), _ptr(m[k] if m else None),
                                                      _ptr(v[k] if v else None), _stream()), lib)
        report(self.verbose, "relocation", [("relocated num", n), ("total gaussian number", N)])
        return dict(relocated=n, total=N)

    @torch.no_grad()
    def grow(self, params, optimizer, generator=None, extra=()):
        """Adds n = max(0, min(cap_max, int(N (1 + grow_rate))) - N) Gaussians drawn by opacity over
        every non-NaN row: rows [0, N) keep their order with the sources updated to their relocation
        value, rows [N, N + n) copy the updated sources in draw order.  Moments are carried, except
        zero for the sources and the new rows.  The Parameters are replaced and the optimizer
        groups / state moved, as DensityController.update_gaussian_density does (a captured
        GraphedFusedStep does not survive this call).  HOST SYNCHRONISATION: one read of the weight
        total.  -> dict(added, total)"""
        lib = _lib.load()
        extra = tuple(extra)
        N, src, m, v, groups = gather_state(params, optimizer, extra, _copy)
        n = max(0, min(self.cap_max, int(N * (1.0 + self.grow_rate))) - N)
        if n:
            ws, w_total, _ = mcmc_plan(src["alphas_raw"], self.alpha_raw_min, MCMC_GROW, n)
            if w_total == 0:
                n = 0
        if n:
            dev = src["pws"].device
            u = torch.rand(n, dtype=torch.float64, device=dev, generator=generator)
            sampled = mcmc_sample(ws, N, u)
            fresh = lambda k: torch.empty((N + n,) + tuple(src[k].shape[1:]), dtype=torch.float32, device=dev)  # noqa: E731
            dst = {k: fresh(k) for k in src}
            dst_m = {k: fresh(k) for k in src} if m is not None else None
            dst_v = {k: fresh(k) for k in src} if m is not None else None
            structs, keep = _structs(src, m, v, dst, dst_m, dst_v)
            _lib.check(lib.gsb_mcmc_grow(N, n, _ptr(sampled), _ptr(ws), ws.numel(), self.min_opacity, self.n_max,
                                         *structs, _stream()), lib)
            for k in extra:
                mk = lambda d: _ptr(d[k] if d is not None else None)  # noqa: E731
                _lib.check(lib.gsb_mcmc_grow_rows(N, n, _ptr(sampled), _ptr(ws), ws.numel(), src[k].shape[1],
                                                  _ptr(src[k]), mk(m), mk(v), _ptr(dst[k]), mk(dst_m), mk(dst_v),
                                                  _stream()), lib)
            swap_parameters(params, optimizer, groups, dst, dst_m, dst_v)
        report(self.verbose, "growth", [("added num", n), ("total gaussian number", N + n)])
        return dict(added=n, total=N + n)

    @torch.no_grad()
    def inject_noise(self, params, optimizer, generator=None):
        """pws += Sigma(q, s) z * lr * noise_lr / (1 + exp(-100 ((1 - o) - 0.995))), in place, with
        z ~ N(0, I) [N, 3] from `generator`, lr the current lr of the "pws" group and Sigma = R S^2 R^T
        of the normalised rots_raw and exp(scales_raw) (no 3D filter, no antialiasing).  Runs after
        optimizer.step(); pointers stay, so a captured GraphedFusedStep stays valid."""
        lib = _lib.load()
        N = params["pws"].shape[0]
        pws = _in_place(params["pws"], "params['pws']", (N, 3))
        a = _check(params["alphas_raw"].detach(), "params['alphas_raw']", (N, 1))
        s = _check(params["scales_raw"].detach(), "params['scales_raw']", (N, 3))
        q = _check(params["rots_raw"].detach(), "params['rots_raw']", (N, 4))
        groups = [g for g in optimizer.param_groups if g.get("name") == "pws"]
        if not groups:
            raise ValueError("the optimizer has no param group named 'pws'")
        lr = float(groups[0]["lr"])
        z = torch.empty((N, 3), dtype=torch.float32, device=pws.device).normal_(0, 1, generator=generator)
        _lib.check(lib.gsb_mcmc_noise(N, _ptr(pws), _ptr(a), _ptr(s), _ptr(q), _ptr(z), lr * self.noise_lr,
                                      self.NOISE_K, self.NOISE_X0, _stream()), lib)
        return z
