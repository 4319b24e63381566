"""Lane-level models of the binning schedule in csrc/binning.cu, checked without a GPU.

* `k_keys`: a warp's 32 Gaussians own one contiguous range of the key array; its lanes walk that
  range 32 positions at a time, find the owning Gaussian by a binary search over the warp's
  exclusive offsets (the shuffle pattern of the kernel) and build the key row-major inside its
  rectangle.  The model must write exactly the keys / ids of the serial per-Gaussian emission of
  the reference (createKeys), each position once, drop a Gaussian that does not fit the capacity
  whole and write nothing at or past the capacity.
* one radix pass: `k_digit_counts` (digit-major counts per sort tile), `k_colscan` (one exclusive
  scan over them, split into CTA spans whose prefixes chain like the decoupled look-back) and the
  scatter of `k_radix_pass` (stable rank inside the tile) must give a stable counting sort, and
  three such passes the (key, id) order of a stable sort.
They say nothing about synchronisation or memory spaces -- that is what the GPU tests are for."""
import numpy as np
import pytest

CS_SPAN = 2048


def serial_keys(n, rects, dks, gx, shift, P):
    """The reference emission: Gaussian by Gaussian, row-major in its rectangle."""
    keys = np.zeros(P, np.uint64)
    vals = np.zeros(P, np.int64)
    pos = 0
    for i in range(len(n)):
        x0, x1, y0, y1 = rects[i]
        for y in range(y0, y1):
            for x in range(x0, x1):
                keys[pos] = ((y * gx + x) << shift) | dks[i]
                vals[pos] = i
                pos += 1
    assert pos == P
    return keys, vals


def warp_keys(n, rects, dks, gx, shift, capacity):
    """k_keys, lane by lane.  Unwritten slots stay -1; returns (keys, vals, status)."""
    N = len(n)
    incl = np.cumsum(n).astype(np.int64)
    P = int(incl[-1]) if N else 0
    keys = np.full(max(P, capacity), -1, np.int64)
    vals = np.full(max(P, capacity), -1, np.int64)
    status = 0
    for first in range(0, N, 32):
        lanes = np.arange(32)
        i = first + lanes
        inc = incl[np.minimum(i, N - 1)]
        off = np.concatenate([[incl[first - 1] if first else 0], inc[:-1]])
        nn = (inc - off).copy()
        drop = (nn > 0) & ((off > capacity) | (nn > capacity - off))
        if drop.any():
            status |= 2
        nn[drop] = 0
        start = off[0]
        span = inc[31] - start
        rel = off - start
        assert np.all(np.diff(rel) >= 0)
        todo = min(span, capacity - start) if start < capacity else 0
        for t0 in range(0, todo, 32):
            for lane in range(32):
                t = t0 + lane
                o = 0
                for s in (16, 8, 4, 2, 1):  # __shfl_sync(rel, o + s) <= t
                    if rel[o + s] <= t:
                        o += s
                local = t - rel[o]
                if t < todo and local < nn[o]:
                    x0, x1, y0, _ = rects[first + o]
                    w = x1 - x0
                    y, x = y0 + local // w, x0 + local % w
                    pos = start + t
                    assert pos < capacity and keys[pos] == -1, "position written twice or past the capacity"
                    keys[pos] = ((y * gx + x) << shift) | dks[first + o]
                    vals[pos] = first + o
    return keys, vals, status


def scene(N, seed, gx=30, gy=20, big=0.05):
    rng = np.random.default_rng(seed)
    rects, n = [], []
    for _ in range(N):
        r = rng.random()
        if r < 0.2:  # culled: no patches
            rects.append((0, 0, 0, 0))
        else:
            w, h = (rng.integers(1, 9), rng.integers(1, 9)) if r < 1 - big else (rng.integers(8, gx), rng.integers(8, gy))
            x0, y0 = rng.integers(0, gx - w + 1), rng.integers(0, gy - h + 1)
            rects.append((x0, x0 + w, y0, y0 + h))
        x0, x1, y0, y1 = rects[-1]
        n.append((x1 - x0) * (y1 - y0))
    dks = rng.integers(0, 1 << 12, N)
    return np.array(n, np.int64), rects, dks


@pytest.mark.parametrize("N,seed", [(1, 0), (31, 1), (32, 2), (33, 3), (200, 4), (1000, 5)])
def test_keys_warp_emission_matches_serial_order(N, seed):
    n, rects, dks = scene(N, seed)
    P = int(n.sum())
    want_k, want_v = serial_keys(n, rects, dks, 30, 12, P)
    got_k, got_v, status = warp_keys(n, rects, dks, 30, 12, capacity=P)
    assert status == 0
    assert np.array_equal(got_k[:P], want_k.astype(np.int64)) and np.array_equal(got_v[:P], want_v)


@pytest.mark.parametrize("N,seed,frac", [(200, 6, 0.5), (1000, 7, 0.9), (1000, 8, 0.0), (64, 9, 0.97)])
def test_keys_capacity_drops_whole_gaussians(N, seed, frac):
    n, rects, dks = scene(N, seed)
    P = int(n.sum())
    cap = int(P * frac)
    want_k, want_v = serial_keys(n, rects, dks, 30, 12, P)
    got_k, got_v, status = warp_keys(n, rects, dks, 30, 12, capacity=cap)
    assert np.all(got_k[cap:] == -1) and np.all(got_v[cap:] == -1)
    off = np.concatenate([[0], np.cumsum(n)[:-1]])
    fits = (n == 0) | ((off <= cap) & (n <= cap - off))
    assert status == (0 if fits.all() else 2)
    for i in np.nonzero(n)[0]:
        sl = slice(off[i], off[i] + n[i])
        if fits[i]:
            assert np.array_equal(got_k[sl], want_k[sl].astype(np.int64)) and np.all(got_v[sl] == i)
        else:
            written = got_v[off[i]:min(off[i] + n[i], cap)]
            assert np.all(written == -1), "a dropped Gaussian was partly written"


def radix_pass(keys, vals, shift, bits, tile):
    """k_digit_counts + k_colscan + k_radix_pass of one LSD pass."""
    P = len(keys)
    bins = 1 << bits
    tiles = (P + tile - 1) // tile
    dig = (keys >> shift) & (bins - 1)
    C = np.zeros((bins, tiles), np.int64)  # digit-major: C[d][t] at d * tiles + t
    for t in range(tiles):
        C[:, t] = np.bincount(dig[t * tile:(t + 1) * tile], minlength=bins)
    flat = C.reshape(-1)
    assert len(flat) % 8 == 0
    B = np.empty_like(flat)  # per CTA span: local exclusive scan + the prefix the look-back hands it
    prefix = 0
    for blk in range(0, len(flat), CS_SPAN):
        span = flat[blk:blk + CS_SPAN]
        B[blk:blk + CS_SPAN] = prefix + np.cumsum(span) - span
        prefix += int(span.sum())
    B = B.reshape(bins, tiles)
    out_k = np.full(P, -1, np.int64)
    out_v = np.full(P, -1, np.int64)
    for t in range(tiles):
        seen = np.zeros(bins, np.int64)
        for j in range(t * tile, min(P, (t + 1) * tile)):  # stable rank inside the tile
            d = dig[j]
            pos = B[d, t] + seen[d]
            seen[d] += 1
            assert out_k[pos] == -1
            out_k[pos], out_v[pos] = keys[j], vals[j]
    return out_k, out_v


@pytest.mark.parametrize("P,bits,tile,seed", [(1, 9, 4096, 0), (5000, 9, 4096, 1), (20000, 9, 4096, 2),
                                              (9000, 8, 2048, 3), (4096, 9, 4096, 4)])
def test_radix_passes_give_a_stable_sort(P, bits, tile, seed):
    rng = np.random.default_rng(seed)
    keys = rng.integers(0, 1 << (3 * bits), P).astype(np.int64)
    keys[rng.random(P) < 0.3] = keys[0]  # many ties: stability decides their order
    vals = np.arange(P, dtype=np.int64)
    k, v = keys, vals
    for p in range(3):
        k, v = radix_pass(k, v, p * bits, bits, tile)
    order = np.argsort(keys, kind="stable")
    assert np.array_equal(k, keys[order]) and np.array_equal(v, vals[order])
