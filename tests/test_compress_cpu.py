"""CPU checks of the compressed export (DESIGN 3.24): the numpy oracle's quantiser and Lloyd step on
hand-made cases, the .npz container written and read back from numpy arrays, every refusal of
load_compressed, the byte count at config-2 scale, and the C ABI's refusals, profile ids and
register use."""
import ctypes as C
import io
import json
import re
import subprocess
import zipfile

import numpy as np
import pytest

from oracle import compress_oracle as co

PTR = 0x10000000


# ----------------------------------------------------------------------------- oracle

def test_oracle_quantiser_hand_made():
    x = np.array([[0.0, 5.0, -1.0], [1.0, 5.0, 0.0], [2.0, 5.0, 1.0], [3.0, 5.0, 3.0]], np.float32)
    q, rng, _ = co.quantize(x, 8)
    assert rng.tolist() == [[0.0, 5.0, -1.0], [3.0, 5.0, 3.0]]
    assert q[:, 0].tolist() == [0, 85, 170, 255]
    assert q[:, 1].tolist() == [0, 0, 0, 0]           # hi == lo: every code 0
    assert q[:, 2].tolist() == [0, 64, 128, 255]      # 63.75 -> 64, 127.5 -> 128 (ties round up)
    assert np.allclose(co.dequantize(q, rng, 8)[:, 0], [0, 1, 2, 3])
    assert (co.dequantize(q, rng, 8)[:, 1] == 5.0).all()
    q16, _, _ = co.quantize(x, 16)
    assert q16[:, 0].tolist() == [0, 21845, 43690, 65535]
    # a caller's range clamps what lies outside it
    q, _, _ = co.quantize(np.array([[-2.0], [0.0], [2.0]], np.float32), 8, value_range=[[-1.0], [1.0]])
    assert q[:, 0].tolist() == [0, 128, 255]


def test_oracle_log_transform_is_odd_and_inverts():
    v = np.array([[-100.0], [-1.0], [0.0], [0.5], [1000.0]], np.float32)
    t = co.transform(v, True)
    assert np.allclose(t[:, 0], np.sign(v[:, 0]) * np.log1p(np.abs(v[:, 0])), rtol=1e-6)
    assert np.allclose(co.inverse_transform(t, True), v, rtol=1e-5)
    q, rng, _ = co.quantize(v, 16, log_transform=True)
    assert q[0, 0] == 0 and q[-1, 0] == 65535
    back = co.dequantize(q, rng, 16, log_transform=True)
    step = (rng[1, 0] - rng[0, 0]) / 65535
    assert np.all(np.abs(co.transform(back.astype(np.float32), True) - t) <= step / 2 + 1e-6)


def test_oracle_boundary_distance():
    assert co.boundary_distance(np.array([0.5, 0.49, 2.0, 1.4999]))[0] == 0.0
    assert np.allclose(co.boundary_distance(np.array([0.49, 2.0, 1.4999])), [0.01, 0.5, 0.0001])


def test_oracle_lloyd_step_hand_made():
    x = np.array([[0.0], [1.0], [10.0], [11.0], [5.0]])
    c = np.array([[0.0], [10.0], [100.0]])
    labels, dmin, gap, _ = co.assign(x, c)
    assert labels.tolist() == [0, 0, 1, 1, 0]          # 5 is 5 from both: the lower index wins
    assert dmin.tolist() == [0, 1, 0, 1, 25] and gap[4] == 0
    new, counts = co.lloyd_update(x, labels, c)
    assert new[:, 0].tolist() == [2.0, 10.5, 100.0]     # the empty cluster keeps its centroid
    assert counts.tolist() == [3, 2, 0]
    assert co.check_assignment(x, c, labels, dmin) == []
    assert co.check_assignment(x, c, [0, 0, 1, 1, 1], dmin) == []       # a tie may go either way
    assert co.check_assignment(x, c, [1, 0, 1, 1, 0], dmin)             # a clear mistake
    assert co.check_assignment(x, c, labels, dmin + 1.0)                # a wrong distance
    t = co.tau(np.array([[3.0, 4.0]]), np.array([[0.0, 0.0], [0.0, 1.0]]))
    assert t[0] == pytest.approx(4 * 2.0 ** -22 * 36)


# ----------------------------------------------------------------------------- container

def _arrays(N, K, seed=0):
    from easygaussiansplatting_b200 import compress as cz
    rng = np.random.default_rng(seed)
    out = {}
    for name, (dt, shape) in cz.ARRAYS.items():
        if name.endswith("_range"):
            lo = rng.uniform(-2, 0, shape(N, K)[1])
            out[name] = np.stack([lo, lo + rng.uniform(0, 3, lo.shape)]).astype(np.float32)
        elif name == "high_shs_labels":
            out[name] = rng.integers(0, K, N).astype(np.uint16)
        else:
            out[name] = rng.integers(0, np.iinfo(dt).max + 1, shape(N, K)).astype(dt)
    return out


def test_container_round_trip(tmp_path):
    from easygaussiansplatting_b200 import compress as cz
    a = _arrays(100, 7)
    p = tmp_path / "scene.gsz"                  # any suffix: the path is used as given
    cz.write_npz(p, a)
    assert p.exists() and not (tmp_path / "scene.gsz.npz").exists()
    back, meta = cz.read_npz(p)
    assert meta == {"format": cz.FORMAT, "version": 1, "N": 100, "K": 7,
                    "bits": {"pws": 16, "scales_raw": 8, "rots_raw": 8, "alphas_raw": 8, "low_shs": 8,
                             "high_shs_codebook": 8},
                    "log_transform": ["pws"]}
    assert sorted(back) == sorted(cz.ARRAYS)
    for k in a:
        assert back[k].dtype == a[k].dtype and (back[k] == a[k]).all(), k
    with zipfile.ZipFile(p) as z:
        assert sorted(z.namelist()) == sorted([k + ".npy" for k in cz.ARRAYS] + ["meta.npy"])
        assert all(i.compress_type == zipfile.ZIP_DEFLATED for i in z.infolist())
    buf = io.BytesIO()
    cz.write_npz(buf, a)
    buf.seek(0)
    assert (cz.read_npz(buf)[0]["pws"] == a["pws"]).all()


def _rewrite(path, arrays, meta=None, drop=()):
    from easygaussiansplatting_b200 import compress as cz
    N, K = arrays["high_shs_labels"].shape[0], arrays["high_shs_codebook"].shape[0]
    m = cz.meta(N, K) if meta is None else meta
    out = {k: v for k, v in arrays.items() if k not in drop}
    out["meta"] = np.frombuffer(json.dumps(m).encode(), np.uint8)
    with open(path, "wb") as f:
        np.savez_compressed(f, **out)


def _refusals(tmp_path):
    """(what, path) of every malformed file load_compressed must refuse"""
    from easygaussiansplatting_b200 import compress as cz
    N, K = 50, 6
    a = _arrays(N, K, seed=1)
    cases = []

    def case(what, **kw):
        p = tmp_path / ("%d.npz" % len(cases))
        kw.setdefault("meta", cz.meta(N, K))
        _rewrite(p, kw.pop("arrays", a), **kw)
        cases.append((what, p))

    case("no 'pws_range' array", drop=("pws_range",))
    case("no 'high_shs_labels' array", drop=("high_shs_labels",))
    case("must be uint16", arrays=dict(a, pws=a["pws"].astype(np.int32)))
    case("must be uint8", arrays=dict(a, high_shs_codebook=a["high_shs_codebook"].astype(np.uint16)))
    case("must be float32", arrays=dict(a, low_shs_range=a["low_shs_range"].astype(np.float64)))
    case("must have shape", arrays=dict(a, rots_raw=a["rots_raw"][:, :3]))
    case("must have shape", arrays=dict(a, scales_raw=a["scales_raw"][:-1]))                 # N disagrees
    case("must have shape", arrays=dict(a, high_shs_codebook=a["high_shs_codebook"][:-1]))   # K disagrees
    case("must have shape", meta=cz.meta(N + 1, K))
    case("must have shape", meta=cz.meta(N, K - 1))
    case("label is >= K", arrays=dict(a, high_shs_labels=np.where(np.arange(N) == 7, K, a["high_shs_labels"])
                                      .astype(np.uint16)))
    case("not finite", arrays=dict(a, pws_range=np.array([[0, 0, np.nan], [1, 1, 1]], np.float32)))
    case("unknown format", meta=dict(cz.meta(N, K), format="spz"))
    case("unknown easygaussiansplatting-compressed version", meta=dict(cz.meta(N, K), version=2))
    case("bit widths", meta=dict(cz.meta(N, K), bits={"pws": 8}))
    case("not 1 <= K", meta=cz.meta(N, 0))
    case("not 1 <= K", meta=cz.meta(K - 1, K))
    p = tmp_path / "nometa.npz"
    np.savez_compressed(p, **a)
    cases.append(("no meta record", p))
    p = tmp_path / "badjson.npz"
    np.savez_compressed(p, meta=np.frombuffer(b"{not json", np.uint8), **a)
    cases.append(("not JSON", p))
    p = tmp_path / "text.npz"
    p.write_bytes(b"ply\nformat ascii 1.0\n")
    cases.append(("", p))
    good = tmp_path / "good.npz"
    _rewrite(good, a)
    p = tmp_path / "truncated.npz"
    p.write_bytes(good.read_bytes()[:len(good.read_bytes()) // 2])
    cases.append(("not a compressed scene file", p))
    p = tmp_path / "pickled.npz"
    obj = dict(a)
    obj["meta"] = np.array([{"format": cz.FORMAT}], dtype=object)
    np.savez(p, **obj)
    cases.append(("pickle", p))
    return cases


def test_load_compressed_refusals(tmp_path):
    from easygaussiansplatting_b200 import compress as cz
    from easygaussiansplatting_b200.gau_io import load_compressed
    for what, p in _refusals(tmp_path):
        with pytest.raises(ValueError, match=re.escape(what) if what else None):
            cz.read_npz(p)
        with pytest.raises(ValueError):
            load_compressed(p, device="cpu")   # refused before anything is decoded
    a = _arrays(5, 5)
    with pytest.raises(ValueError, match="label is >= K"):
        cz.write_npz(tmp_path / "w.npz", dict(a, high_shs_labels=np.full(5, 9, np.uint16)))


def test_byte_accounting_at_config2_scale(tmp_path):
    from easygaussiansplatting_b200 import compress as cz
    N, K = 1_000_000, 65536
    payload = cz.payload_bytes(N, K)
    assert payload == 19 * N + 45 * K                    # 21.9 MB
    assert 248 * N / payload > 11                         # save_ply writes 62 float32 columns
    a = _arrays(N, K, seed=2)                             # uniform random codes: deflate gains nothing
    p = tmp_path / "big.npz"
    cz.write_npz(p, a)
    size = p.stat().st_size
    assert size <= 1.01 * payload + 64 * 1024, (size, payload)


# ----------------------------------------------------------------------------- C ABI

def _lib():
    from easygaussiansplatting_b200 import _lib as L, build
    build.build()
    return L, L.load()


def test_entry_points_refuse_bad_arguments_before_any_launch():
    L, lib = _lib()
    vp = C.c_void_p
    assert lib.gsb_kmeans_assign_workspace_bytes(65536, 45) == 46 * 65536 * 4
    assert lib.gsb_kmeans_assign_workspace_bytes(1, 1) == 2 * 128 * 4
    assert lib.gsb_kmeans_assign_workspace_bytes(129, 3) == 4 * 256 * 4
    for K, D in ((0, 3), (1, 0), (1, 65), (2 ** 31 - 127, 3)):
        assert lib.gsb_kmeans_assign_workspace_bytes(K, D) == 0

    def assign(N=10, K=4, D=3, x=PTR, ldx=3, c=PTR, labels=PTR, dist=PTR, ws=PTR, ws_bytes=1 << 20):
        rc = lib.gsb_kmeans_assign(N, K, D, vp(x), ldx, vp(c), vp(labels), vp(dist), vp(ws), ws_bytes, None)
        return rc, lib.gsb_last_error().decode()

    for kw, text in [({"N": -1}, "N < 0"), ({"K": 0}, "K < 1"), ({"D": 0}, "D out of [1, 64]"),
                     ({"D": 65}, "D out of [1, 64]"), ({"K": 2 ** 31 - 127}, "K overflows the centroid index"),
                     ({"ldx": 2}, "ldx < D"), ({"N": 3, "ldx": 2 ** 62}, "N ldx overflows"),
                     ({"x": None}, "null pointer"), ({"c": None}, "null pointer"), ({"ws": None}, "null pointer"),
                     ({"labels": None}, "null pointer"), ({"x": PTR + 2}, "misaligned"),
                     ({"dist": PTR + 1}, "misaligned"), ({"ws": PTR + 4}, "misaligned"),
                     ({"ws_bytes": 4 * 128 * 4 - 1}, "workspace too small")]:
        rc, msg = assign(**kw)
        assert rc == -1 and "kmeans_assign: " + text in msg, (kw, msg)
    assert assign(N=0, x=None, labels=None, dist=None)[0] == 0        # nothing to assign: no launch

    def update(N=10, K=4, D=3, x=PTR, ldx=3, labels=PTR, perm=PTR, c=PTR, out=PTR, counts=PTR):
        rc = lib.gsb_kmeans_update(N, K, D, vp(x), ldx, vp(labels), vp(perm), vp(c), vp(out), vp(counts), None)
        return rc, lib.gsb_last_error().decode()

    for kw, text in [({"N": -1}, "N < 0"), ({"K": 0}, "K < 1"), ({"D": 65}, "D out of [1, 64]"),
                     ({"ldx": 1}, "ldx < D"), ({"perm": None}, "null pointer"), ({"counts": None}, "null pointer"),
                     ({"out": None}, "null pointer"), ({"perm": PTR + 2}, "misaligned"),
                     ({"x": PTR + 1}, "misaligned")]:
        rc, msg = update(**kw)
        assert rc == -1 and "kmeans_update: " + text in msg, (kw, msg)

    def quant(N=10, D=3, x=PTR, ldx=3, bits=8, log_t=0, fit=1, rng=PTR, codes=PTR):
        rc = lib.gsb_quantize(N, D, vp(x), ldx, bits, log_t, fit, vp(rng), vp(codes), None)
        return rc, lib.gsb_last_error().decode()

    for kw, text in [({"N": -1}, "N < 0"), ({"D": 0}, "D out of [1, 64]"), ({"bits": 12}, "bits must be 8 or 16"),
                     ({"ldx": 2}, "ldx < D"), ({"rng": None}, "null pointer"), ({"codes": None}, "null pointer"),
                     ({"bits": 16, "codes": PTR + 1}, "misaligned"), ({"x": PTR + 2}, "misaligned")]:
        rc, msg = quant(**kw)
        assert rc == -1 and "quantize: " + text in msg, (kw, msg)

    def dequant(N=10, D=3, codes=PTR, bits=8, rng=PTR, log_t=0, out=PTR):
        rc = lib.gsb_dequantize(N, D, vp(codes), bits, vp(rng), log_t, vp(out), None)
        return rc, lib.gsb_last_error().decode()

    for kw, text in [({"N": -1}, "N < 0"), ({"D": 65}, "D out of [1, 64]"), ({"bits": 32}, "bits must be 8 or 16"),
                     ({"out": None}, "null pointer"), ({"bits": 16, "codes": PTR + 1}, "misaligned"),
                     ({"out": PTR + 2}, "misaligned")]:
        rc, msg = dequant(**kw)
        assert rc == -1 and "dequantize: " + text in msg, (kw, msg)
    assert dequant(N=0, codes=None, rng=None, out=None)[0] == 0
    assert lib.gsb_abi_version() == 1


def test_signatures_profile_ids_and_register_use():
    L, lib = _lib()
    for name in ("gsb_kmeans_assign_workspace_bytes", "gsb_kmeans_assign", "gsb_kmeans_update", "gsb_quantize",
                 "gsb_dequantize"):
        assert name in L.SIGNATURES and hasattr(lib, name), name
    names = [lib.gsb_profile_kernel_name(i).decode() for i in range(lib.gsb_profile_kernels())]
    i = names.index("draw_backward_rgbd_batch")
    assert names[i + 1:i + 6] == ["kmeans_assign", "kmeans_update", "quantize", "dequantize", "density_apply_rows"]
    sass = subprocess.run(["cuobjdump", "-sass", L.LIB_PATH], capture_output=True, text=True).stdout
    body = [f for f in re.split(r"\n\s*Function : ", sass) if "15k_kmeans_assign" in f.split("\n")[0]]
    assert len(body) == 1
    for op in ("LDGSTS.E.BYPASS.128", "LDGDEPBAR", "DEPBAR.LE", "LDS.128", "FFMA"):
        assert op in body[0], op
    r = subprocess.run(["cuobjdump", "-res-usage", L.LIB_PATH], capture_output=True, text=True)
    found = dict(re.findall(r"Function (\S*(?:k_kmeans_\w+|k_quant\w*|k_dequantize\w*)):\s*\n\s*(REG:.*)", r.stdout))
    assert len(found) == 9, sorted(found)
    for name, usage in found.items():
        assert "LOCAL:0 " in usage and "STACK:0 " in usage, (name, usage)
        if "k_kmeans_assign" in name:
            assert int(re.search(r"REG:(\d+)", usage).group(1)) <= 128, usage   # two 256-thread CTAs per SM
