"""CPU oracle for MCMC densification (Kheradmand et al. 2024; DESIGN 3.11).  TEST INFRASTRUCTURE
ONLY -- imported by tests/ (and nothing in the product).

- The sampler is exact integer arithmetic: weights floor(o 2^32) in uint64, their prefix sum and
  the search are the kernels' operations, so sample ids agree id for id.
- The relocation value is evaluated in np.longdouble (the kernels use fp64) and rounded to fp32
  once.
- The noise displacement is fp64 on the fp32 inputs, with the quaternion conventions of
  density_oracle._normalize / _rotate: (w, x, y, z), q / max(|q|, 1e-12).
"""
import numpy as np

from . import density_oracle as dor

F = np.float32
NAMES = dor.NAMES
L = np.longdouble


def alpha_raw_min(min_opacity=0.005):
    """the fp32 logit the kernels compare alphas_raw with (density.raw_thresholds' arithmetic)"""
    return F(np.log(min_opacity / (1 - min_opacity)))


def dead_rows(alphas_raw, min_opacity=0.005):
    """ascending ids of the rows with !(alphas_raw > logit(min_opacity)), NaN included"""
    a = np.asarray(alphas_raw, F).reshape(-1)
    with np.errstate(invalid="ignore"):
        return np.flatnonzero(~(a > alpha_raw_min(min_opacity)))


def weights(alphas_raw, mode, min_opacity=0.005):
    """uint64 q_i = floor(o_i 2^32), o_i = sigmoid in fp64; 0 for NaN rows and, in mode "relocate",
    for dead rows"""
    a = np.asarray(alphas_raw, F).reshape(-1)
    with np.errstate(over="ignore", invalid="ignore"):
        o = 1.0 / (1.0 + np.exp(-a.astype(np.float64)))
        q = np.floor(o * 4294967296.0)
    q[np.isnan(a)] = 0
    if mode == "relocate":
        q[dead_rows(a, min_opacity)] = 0
    return q.astype(np.uint64)


def sample(w, u):
    """ids of the draws u[n] (fp64 in [0, 1)) under integer weights w: the first i with
    W_i > min(floor(u W_total), W_total - 1), W the inclusive prefix sum"""
    W = np.cumsum(w.astype(np.uint64), dtype=np.uint64)
    total = int(W[-1]) if len(W) else 0
    assert total > 0
    t = np.floor(np.asarray(u, np.float64) * np.float64(total))
    t = np.minimum(t.astype(np.uint64), np.uint64(total - 1))
    return np.searchsorted(W, t, side="right").astype(np.int64)


def series(op, r):
    """sum_{m=1..r} C(r,m) (-1)^(m+1) op^m / sqrt(m) in np.longdouble"""
    op = L(op)
    s, binom = L(0), L(1)
    for m in range(1, r + 1):
        binom = binom * L(r - m + 1) / L(m)
        term = binom * op ** m / np.sqrt(L(m))
        s += term if m % 2 else -term
    return s


def new_opacity(o, om, r, min_opacity=0.005):
    """(o', 1 - o') in np.longdouble from o and om = 1 - o, each computed on its own:
    o' = clamp(1 - om^(1/r), min_opacity, 1 - 2^-23), and o' = o for r = 1"""
    o, om = L(o), L(om)
    op, q = (o, om) if r == 1 else (L(1) - om ** (L(1) / L(r)), om ** (L(1) / L(r)))
    if op < L(min_opacity):
        return L(min_opacity), L(1) - L(min_opacity)
    if q < L(2) ** -23:
        return L(1) - L(2) ** -23, L(2) ** -23
    return op, q


def relocation_value(alpha_raw, scale_raw, c, min_opacity=0.005, n_max=51):
    """(alphas_raw', scales_raw'[3]) of a source hit c times, each rounded to fp32 once"""
    r = min(c + 1, n_max)
    a = L(float(F(alpha_raw)))
    o, om = L(1) / (L(1) + np.exp(-a)), L(1) / (L(1) + np.exp(a))
    op, q = new_opacity(o, om, r, min_opacity)
    f = np.log(o / series(op, r))
    s = np.array([F(L(float(F(x))) + f) for x in np.asarray(scale_raw).reshape(-1)], F)
    return F(np.log(op / q)), s


def _update_sources(params, sampled, min_opacity, n_max):
    """params with every sampled source's alphas_raw / scales_raw replaced by its relocation value"""
    out = {k: np.array(v, F, copy=True) for k, v in params.items()}
    ids, cnt = np.unique(sampled, return_counts=True)
    for i, c in zip(ids, cnt):
        a, s = relocation_value(params["alphas_raw"].reshape(-1)[i], params["scales_raw"][i], int(c),
                                min_opacity, n_max)
        out["alphas_raw"].reshape(-1)[i] = a
        out["scales_raw"][i] = s
    return out


def relocate(params, m, v, u, min_opacity=0.005, n_max=51):
    """in-place relocation of the dead rows.  params / m / v: dicts of [N, w] arrays (the six names
    and any extra ones; m, v None = no optimizer state).  u: fp64 uniforms, one per dead row.
    -> (params', m', v', dead ids, sampled ids)"""
    dead = dead_rows(params["alphas_raw"], min_opacity)
    w = weights(params["alphas_raw"], "relocate", min_opacity)
    if len(dead) == 0 or int(w.sum(dtype=np.uint64)) == 0:
        return params, m, v, dead[:0], dead[:0]
    sampled = sample(w, u[: len(dead)])
    out = _update_sources(params, sampled, min_opacity, n_max)
    for k in out:
        out[k][dead] = out[k][sampled]
    mo = vo = None
    if m is not None:
        mo = {k: np.array(x, F, copy=True) for k, x in m.items()}
        vo = {k: np.array(x, F, copy=True) for k, x in v.items()}
        for d in (mo, vo):
            for k in d:
                d[k][sampled] = 0
                d[k][dead] = 0
    return out, mo, vo, dead, sampled


def grow_count(N, cap_max, grow_rate=0.05):
    """n = max(0, min(cap_max, int(N (1 + grow_rate))) - N)"""
    return max(0, min(cap_max, int(N * (1.0 + grow_rate))) - N)


def grow(params, m, v, u, n, min_opacity=0.005, n_max=51):
    """[N + n] tensors: the rows with the sources updated, then copies of the updated sources in draw
    order; moments carried except zero for the sources and the new rows.  -> (params', m', v',
    sampled ids)"""
    w = weights(params["alphas_raw"], "grow", min_opacity)
    sampled = sample(w, u[:n])
    upd = _update_sources(params, sampled, min_opacity, n_max)
    out = {k: np.concatenate([upd[k], upd[k][sampled]]) for k in upd}
    mo = vo = None
    if m is not None:
        mo, vo = {}, {}
        for src, dst in ((m, mo), (v, vo)):
            for k, x in src.items():
                x = np.array(x, F, copy=True)
                x[sampled] = 0
                dst[k] = np.concatenate([x, np.zeros((n,) + x.shape[1:], F)])
    return out, mo, vo, sampled


def noise(params, z, lr, noise_lr=5e5, k=100.0, x0=float(F(0.995))):
    """the displacement Sigma(q, s) z lr noise_lr / (1 + exp(-k ((1 - o) - x0))) in fp64; x0 defaults
    to the fp32 value the kernel is given"""
    a = np.asarray(params["alphas_raw"], np.float64).reshape(-1)
    s = np.exp(np.asarray(params["scales_raw"], np.float64))
    q = np.asarray(params["rots_raw"], np.float64)
    q = q / np.maximum(np.sqrt((q * q).sum(axis=1)), 1e-12)[:, None]
    w, x, y, zq = q.T
    R = np.stack([1 - 2 * (y * y + zq * zq), 2 * (x * y - zq * w), 2 * (x * zq + y * w),
                  2 * (x * y + zq * w), 1 - 2 * (x * x + zq * zq), 2 * (y * zq - x * w),
                  2 * (x * zq - y * w), 2 * (y * zq + x * w), 1 - 2 * (x * x + y * y)], axis=1).reshape(-1, 3, 3)
    M = R * s[:, None, :]
    Sigma = M @ M.transpose(0, 2, 1)
    with np.errstate(over="ignore"):
        gate = 1.0 / (1.0 + np.exp(-k * (1.0 / (1.0 + np.exp(a)) - x0)))
    return np.einsum("nij,nj->ni", Sigma, np.asarray(z, np.float64)) * (lr * noise_lr * gate)[:, None]
