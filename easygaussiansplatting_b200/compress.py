"""Compressed scene export (DESIGN 3.24): gsplat's `--compression` scheme without the PNG container
and the PLAS sort.  The 45 higher-order SH coefficients of each Gaussian are vector-quantised
against a k-means codebook (ops.kmeans_assign / ops.kmeans_update, CUDA), and every other attribute
is stored as 8 or 16-bit codes with a per-column range (ops.quantize, CUDA):

    tensor        stored as                                             bytes / Gaussian
    pws           sign(v) log1p(|v|), per-axis 16-bit                   6
    scales_raw    per-column 8-bit                                      3
    rots_raw      normalised, then [-1, 1] -> 8-bit                     4
    alphas_raw    8-bit                                                 1
    low_shs       per-column 8-bit                                      3
    high_shs      codebook label, uint16 (so K <= 65536)                2
    codebook      [K, 45], per-column 8-bit                             45 K in total

    enc = compress(params)             # dict of device tensors (ARRAYS)
    params = decompress(enc)           # the six raw training tensors

`write_npz` / `read_npz` are the file: one np.savez_compressed archive of those arrays and a JSON
`meta` array, read back without pickles and checked before anything is decoded
(gau_io.save_compressed / load_compressed put the two halves together).
"""
import json
import zipfile

import numpy as np
import torch

from . import ops
from ._lib import GAUSSIAN_TENSORS, GAUSSIAN_WIDTHS

FORMAT = "easygaussiansplatting-compressed"
VERSION = 1
MAX_CLUSTERS = 65536
SH_DIM = 45

# name -> (numpy dtype, shape as a function of (N, K)); the codes and the fp32 ranges of the file
ARRAYS = {
    "pws": (np.uint16, lambda N, K: (N, 3)),
    "pws_range": (np.float32, lambda N, K: (2, 3)),
    "scales_raw": (np.uint8, lambda N, K: (N, 3)),
    "scales_raw_range": (np.float32, lambda N, K: (2, 3)),
    "rots_raw": (np.uint8, lambda N, K: (N, 4)),
    "rots_raw_range": (np.float32, lambda N, K: (2, 4)),
    "alphas_raw": (np.uint8, lambda N, K: (N, 1)),
    "alphas_raw_range": (np.float32, lambda N, K: (2, 1)),
    "low_shs": (np.uint8, lambda N, K: (N, 3)),
    "low_shs_range": (np.float32, lambda N, K: (2, 3)),
    "high_shs_labels": (np.uint16, lambda N, K: (N,)),
    "high_shs_codebook": (np.uint8, lambda N, K: (K, SH_DIM)),
    "high_shs_range": (np.float32, lambda N, K: (2, SH_DIM)),
}
# tensor -> (bits, log transform) of its scalar codes
BITS = {"pws": (16, True), "scales_raw": (8, False), "rots_raw": (8, False), "alphas_raw": (8, False),
        "low_shs": (8, False), "high_shs_codebook": (8, False)}


def payload_bytes(N, K):
    """the bytes of the codes alone: 19 N + 45 K"""
    return sum(np.dtype(dt).itemsize * int(np.prod(shape(N, K))) for name, (dt, shape) in ARRAYS.items()
               if not name.endswith("_range"))


def kmeans(x, K, iters=10, init=None, generator=None):
    """Lloyd's k-means of the rows of x[N, D] (float32 CUDA, 1 <= D <= 64) with K = min(K, N)
    clusters.  init: None (K distinct rows drawn with `generator`, a torch.Generator on x's device, or
    torch's default one) or the starting centroids [K, D].  Each iteration assigns every row to its
    nearest centroid (ops.kmeans_assign) and moves the centroids to the means of their rows
    (ops.kmeans_update); a final assignment follows the last update.
    -> (centroids [K, D], labels int32 [N], distortion float64 [iters + 1]: the mean squared distance
    after each assignment, on the host)"""
    if not isinstance(x, torch.Tensor) or x.dim() != 2:
        raise ValueError("x must be an [N, D] tensor")
    N = x.shape[0]
    if N < 1:
        raise ValueError("k-means needs at least one row")
    if int(iters) < 0:
        raise ValueError("iters must be >= 0")
    if init is None:
        K = min(int(K), N)
        if K < 1:
            raise ValueError("K must be >= 1")
        pick = torch.randperm(N, generator=generator, device=x.device)[:K]
        centroids = x[pick].contiguous()
    else:
        centroids = init.detach().to(torch.float32).contiguous()
        if centroids.dim() != 2 or centroids.shape[1] != x.shape[1] or not 1 <= centroids.shape[0] <= N:
            raise ValueError("init must be [K, %d] with 1 <= K <= N, got %s" % (x.shape[1], tuple(centroids.shape)))
    distortion = []
    labels, dist = ops.kmeans_assign(x, centroids)
    distortion.append(dist.double().mean())
    for _ in range(int(iters)):
        centroids, _counts = ops.kmeans_update(x, labels, centroids)
        labels, dist = ops.kmeans_assign(x, centroids)
        distortion.append(dist.double().mean())
    return centroids, labels, torch.stack(distortion).cpu().numpy()


def compress(params, sh_clusters=65536, iters=10, generator=None):
    """The encoded model of the six raw training tensors `params` (float32 CUDA, N >= 1 rows):
    a dict with the keys of ARRAYS as device tensors (uint16 codes as torch.uint16).  The SH
    codebook has min(sh_clusters, N) rows; with sh_clusters >= N the SH rows are only scalar
    quantised (every row is its own centroid)."""
    if not 1 <= int(sh_clusters) <= MAX_CLUSTERS:
        raise ValueError("sh_clusters must be in [1, %d] (uint16 labels), got %r" % (MAX_CLUSTERS, sh_clusters))
    src = {}
    for k, w in zip(GAUSSIAN_TENSORS, GAUSSIAN_WIDTHS):
        t = params[k].detach()
        if t.dim() != 2 or t.shape[1] != w:
            raise ValueError("params[%r] must be [N, %d], got %s" % (k, w, tuple(t.shape)))
        src[k] = t
    N = src["pws"].shape[0]
    if any(t.shape[0] != N for t in src.values()):
        raise ValueError("the six training tensors disagree on N")
    if N < 1:
        raise ValueError("there is nothing to compress (N = 0)")
    enc = {}
    for k in ("pws", "scales_raw", "alphas_raw", "low_shs"):
        bits, log_t = BITS[k]
        enc[k], enc[k + "_range"] = ops.quantize(src[k], bits, log_transform=log_t)
    rots = src["rots_raw"] / src["rots_raw"].norm(dim=1, keepdim=True)
    unit = torch.tensor([[-1.0] * 4, [1.0] * 4], dtype=torch.float32, device=rots.device)
    enc["rots_raw"], enc["rots_raw_range"] = ops.quantize(rots, 8, value_range=unit)
    codebook, labels, _ = kmeans(src["high_shs"], sh_clusters, iters=iters, generator=generator)
    enc["high_shs_labels"] = labels.to(torch.uint16)
    enc["high_shs_codebook"], enc["high_shs_range"] = ops.quantize(codebook, 8)
    return enc


def decompress(encoded):
    """The six raw training tensors (float32, on the device of the codes) of compress's output"""
    out = {}
    for k in ("pws", "scales_raw", "rots_raw", "alphas_raw", "low_shs"):
        out[k] = ops.dequantize(encoded[k], encoded[k + "_range"], log_transform=BITS[k][1])
    codebook = ops.dequantize(encoded["high_shs_codebook"], encoded["high_shs_range"])
    out["high_shs"] = codebook[encoded["high_shs_labels"].to(torch.int64)]
    return {k: out[k] for k in GAUSSIAN_TENSORS}


def meta(N, K):
    """the file's meta record"""
    return {"format": FORMAT, "version": VERSION, "N": int(N), "K": int(K),
            "bits": {k: b for k, (b, _) in BITS.items()}, "log_transform": [k for k, (_, t) in BITS.items() if t]}


def write_npz(f, arrays):
    """Writes the numpy arrays of ARRAYS (checked as read_npz checks them) and the meta record to
    f (a path or a binary file) as one np.savez_compressed archive; a path is used as given."""
    N, K = arrays["high_shs_labels"].shape[0], arrays["high_shs_codebook"].shape[0]
    out = _checked(arrays, N, K)
    out["meta"] = np.frombuffer(json.dumps(meta(N, K), sort_keys=True).encode("utf-8"), np.uint8)
    if isinstance(f, (str, bytes)) or hasattr(f, "__fspath__"):
        with open(f, "wb") as fh:
            np.savez_compressed(fh, **out)
    else:
        np.savez_compressed(f, **out)


def read_npz(f):
    """-> (dict of the numpy arrays of ARRAYS, meta dict).  Reads without pickles and raises
    ValueError on an unknown format or version, a missing array, a wrong dtype or shape, N or K that
    disagree between the arrays and the meta record, a label >= K, or a non-finite range."""
    try:
        with np.load(f, allow_pickle=False) as z:  # a file that is not an archive raises ValueError here
            files = {k: z[k] for k in z.files}
    except (OSError, EOFError, zipfile.BadZipFile) as e:
        raise ValueError("not a compressed scene file: %s" % e)
    if "meta" not in files or files["meta"].dtype != np.uint8 or files["meta"].ndim != 1:
        raise ValueError("the file has no meta record")
    try:
        m = json.loads(files["meta"].tobytes().decode("utf-8"))
    except (UnicodeDecodeError, json.JSONDecodeError) as e:
        raise ValueError("the meta record is not JSON: %s" % e)
    if not isinstance(m, dict) or m.get("format") != FORMAT:
        raise ValueError("unknown format %r" % (m.get("format") if isinstance(m, dict) else m,))
    if m.get("version") != VERSION:
        raise ValueError("unknown %s version %r" % (FORMAT, m.get("version")))
    N, K = m.get("N"), m.get("K")
    if not (isinstance(N, int) and isinstance(K, int) and N >= 1 and 1 <= K <= min(N, MAX_CLUSTERS)):
        raise ValueError("meta N = %r, K = %r are not 1 <= K <= min(N, %d)" % (N, K, MAX_CLUSTERS))
    if m != meta(N, K):
        raise ValueError("the meta record's bit widths or transforms are not version %d's" % VERSION)
    return _checked(files, N, K), m


def _checked(arrays, N, K):
    out = {}
    for name, (dt, shape) in ARRAYS.items():
        if name not in arrays:
            raise ValueError("the file has no %r array" % name)
        a = np.asarray(arrays[name])
        if a.dtype != np.dtype(dt):
            raise ValueError("%r must be %s, got %s" % (name, np.dtype(dt), a.dtype))
        if a.shape != shape(N, K):
            raise ValueError("%r must have shape %s for N = %d, K = %d, got %s" % (name, shape(N, K), N, K, a.shape))
        if name.endswith("_range") and not np.isfinite(a).all():
            raise ValueError("%r is not finite" % name)
        out[name] = a
    if len(out["high_shs_labels"]) and int(out["high_shs_labels"].max()) >= K:
        raise ValueError("a high_shs label is >= K = %d" % K)
    return out


def to_numpy(encoded):
    """compress's device tensors -> host numpy arrays of ARRAYS' dtypes"""
    return {k: encoded[k].cpu().numpy() for k in ARRAYS}


def to_device(arrays, device="cuda"):
    """read_npz's arrays -> the device tensors decompress takes"""
    return {k: torch.from_numpy(np.ascontiguousarray(a)).to(device) for k, a in arrays.items()}
