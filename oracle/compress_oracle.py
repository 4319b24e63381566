"""fp64 / numpy model of the compressed export (DESIGN 3.24; easygaussiansplatting_b200/csrc/compress.cu):
the scalar quantiser and its inverse, the nearest-centroid assignment with its accuracy contract, and
one Lloyd update."""
import numpy as np


def transform(v, log_transform):
    """sign(v) log1p(|v|) (positions) or v, in float32 as the kernels compute it"""
    v = np.asarray(v, np.float32)
    return np.copysign(np.log1p(np.abs(v)), v).astype(np.float32) if log_transform else v


def inverse_transform(y, log_transform):
    y = np.asarray(y, np.float64)
    return np.copysign(np.expm1(np.abs(y)), y) if log_transform else y


def fit_range(x, log_transform=False):
    """[2, D] float32: each column's min and max of the transformed values"""
    t = transform(x, log_transform)
    return np.stack([t.min(axis=0), t.max(axis=0)]).astype(np.float32)


def quantize(x, bits, log_transform=False, value_range=None):
    """-> (codes int64 [N, D], range float32 [2, D], r float64 [N, D]) with
    q = clamp(floor(r + 1/2), 0, 2^bits - 1), r = (t - lo) (2^bits - 1) / (hi - lo) in fp64
    (hi == lo: q = 0, r = 0).  r tells how near a code is to a rounding boundary."""
    t = transform(x, log_transform).astype(np.float64)
    rng = fit_range(x, log_transform) if value_range is None else np.asarray(value_range, np.float32)
    lo, hi = rng[0].astype(np.float64), rng[1].astype(np.float64)
    qmax = float(2 ** bits - 1)
    span = hi - lo
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(span > 0, (t - lo) * qmax / np.where(span > 0, span, 1.0), 0.0)
    q = np.clip(np.floor(r + 0.5), 0, qmax).astype(np.int64)
    return q, rng, r


def boundary_distance(r):
    """how far r + 1/2 is from the nearest integer: codes may differ by one where this is tiny"""
    s = r + 0.5
    return np.abs(s - np.round(s))


def dequantize(codes, value_range, bits, log_transform=False):
    rng = np.asarray(value_range, np.float64)
    v = rng[0] + np.asarray(codes, np.float64) * (rng[1] - rng[0]) / float(2 ** bits - 1)
    return inverse_transform(v, log_transform)


def distances(x, c):
    """fp64 squared distances [N, K]"""
    x = np.asarray(x, np.float64)
    c = np.asarray(c, np.float64)
    return ((x[:, None, :] - c[None, :, :]) ** 2).sum(axis=2)


def tau(x, c):
    """the assignment's tolerance per point: (D + 2) 2^-22 (|x| + max_k |c_k|)^2"""
    x = np.asarray(x, np.float64)
    c = np.asarray(c, np.float64)
    cmax = np.sqrt((c * c).sum(axis=1)).max()
    return (x.shape[1] + 2) * 2.0 ** -22 * (np.sqrt((x * x).sum(axis=1)) + cmax) ** 2


def assign(x, c):
    """-> (labels: the fp64 argmin, lowest index on ties; the nearest distance; the gap from the
    nearest to the runner-up (inf for K = 1); the full distance matrix)"""
    d = distances(x, c)
    labels = np.argmin(d, axis=1)
    dmin = d[np.arange(len(d)), labels]
    if d.shape[1] > 1:
        part = np.partition(d, 1, axis=1)
        gap = part[:, 1] - part[:, 0]
    else:
        gap = np.full(len(d), np.inf)
    return labels, dmin, gap, d


def check_assignment(x, c, labels, dist):
    """The accuracy contract of gsb_kmeans_assign: with tau as above,
      d(x, c_label) - min_k d(x, c_k) <= tau,
      label == the fp64 argmin wherever the fp64 gap to the runner-up exceeds tau,
      |dist - d(x, c_label)| <= tau.
    -> list of violation messages (empty when the contract holds)"""
    ref, dmin, gap, d = assign(x, c)
    t = tau(x, c)
    labels = np.asarray(labels, np.int64)
    bad = []
    if labels.min(initial=0) < 0 or labels.max(initial=0) >= c.shape[0]:
        return ["labels outside [0, K)"]
    got = d[np.arange(len(d)), labels]
    excess = got - dmin
    if (excess > t).any():
        bad.append("%d labels farther than tau from the nearest" % int((excess > t).sum()))
    clear = gap > t
    if (labels[clear] != ref[clear]).any():
        bad.append("%d clear labels differ from the fp64 argmin" % int((labels[clear] != ref[clear]).sum()))
    derr = np.abs(np.asarray(dist, np.float64) - got)
    if (derr > t).any():
        bad.append("%d distances off by more than tau" % int((derr > t).sum()))
    return bad


def lloyd_update(x, labels, c):
    """-> (new centroids fp64 [K, D], counts [K]): the mean of each cluster's members; an empty
    cluster keeps its centroid"""
    x = np.asarray(x, np.float64)
    c = np.asarray(c, np.float64)
    K = c.shape[0]
    labels = np.asarray(labels, np.int64)
    counts = np.bincount(labels, minlength=K)
    sums = np.zeros_like(c)
    np.add.at(sums, labels, x)
    out = c.copy()
    nz = counts > 0
    out[nz] = sums[nz] / counts[nz, None]
    return out, counts
