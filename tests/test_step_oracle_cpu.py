"""CPU checks of the fp64 whole-step oracle (oracle/step_oracle.py), the reference every fused training
step is held to in test_gpu_step_matrix.py: with every flag off it is the colour chain the end-to-end
test has always used, with one flag on it is the composition that flag's own tests do, bit for bit in
fp64; and with all four flags on its gradients -- the Gaussians' and the camera's -- agree with central
differences of L = <dl, image> + <dld, D> + <dla, A> through the composed forward."""
import numpy as np
import pytest

from oracle import filter3d_oracle as of3
from oracle import oracle as orc
from oracle import pose_oracle as opose
from oracle import rgbd_oracle as ordb
from oracle import step_oracle as ost
from easygaussiansplatting_b200.scene import upstream_gradient

from test_antialias_cpu import H, W, edge_scene, oracle_backward
from test_filter3d_cpu import camera_row, ring_table
from test_fused_math_cpu import _scene

K3 = 4


def _case(n=2000, k3=K3, seed=31):
    sc, rows = edge_scene(k3, seed=seed, n=n)
    rng = np.random.default_rng(seed + 1)
    sc["alphas"] = rng.uniform(0.05, 1.0, n).astype(np.float32)
    dl = upstream_gradient(W, H, seed) * np.float32(3.0 * W * H)
    dld = (rng.normal(size=(H, W)) * 0.3).astype(np.float32)
    dla = rng.normal(size=(H, W)).astype(np.float32)
    return sc, rows, dl, dld, dla


def _filter(sc, Wf=W, Hf=H, seed=3):
    """the oracle filter of a few ring cameras plus the render camera, as the GPU tests pass it (fp32)"""
    table = np.concatenate([ring_table(4, seed=seed),
                            camera_row(sc["Rcw"], sc["tcw"], sc["fx"], sc["fy"], sc["cx"], sc["cy"], Wf, Hf)[None]])
    return of3.filter3d(sc["pws"], table)["filter"].astype(np.float32)


@pytest.fixture
def serial():
    """one OpenMP thread: the oracle's rasterizer backward sums per Gaussian with `omp atomic` under a
    dynamic schedule, so only a serial run gives the same fp64 bits twice"""
    n = orc.num_threads()
    orc.set_num_threads(1)
    yield
    orc.set_num_threads(n)


def _eq(a, b, name):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64).reshape(np.shape(a))
    assert np.array_equal(a, b), (name, np.abs(a - b).max())


def _step(sc, dl, dld=None, dla=None, filt=None, **flags):
    kw = dict(rgbd=False, pose=False, aa=False)
    kw.update(flags)
    return ost.step(sc, ost.camera(sc, W, H), filt=filt, dl=dl, dld=dld, dla=dla, **kw)


# ---------------------------------------------------------------- each flag is its own tests' composition
def test_all_flags_off_is_the_colour_chain(serial):
    sc, _, dl, _, _ = _case()
    got = _step(sc, dl)
    st = opose.stages(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                      sc["fy"], sc["cx"], sc["cy"], W, H)
    fwd = orc.splat(H, W, st["us"], st["ci"], sc["alphas"], st["depths"].copy(), st["col"], st["areas"].copy())
    du, dc, da, dcol, amb = orc.splat_backward(H, W, st["us"], st["ci"], sc["alphas"], st["col"], fwd, dl,
                                               return_ambiguous=True)
    ref = orc.chain_backward(sc["Rcw"], du, dc, da, dcol, *st["J"])
    _eq(got["image"], fwd["image"], "image")
    assert got["depth"] is None and got["alpha"] is None
    for k in ("pws", "shs", "scales", "rots", "alphas", "us"):
        _eq(got["grads"][k], ref[k], k)
    assert not got["per"].any()
    assert np.array_equal(got["flagged"], amb | got["band"] | got["thin"])
    assert got["thin"][4:8].all() and got["thin_pixels"].any()  # edge_scene's needles
    assert amb.any() and fwd["P"] > 0  # (the scene reaches the rasterizer's threshold band)


def test_aa_alone_is_oracle_backward(serial):
    """test_antialias_cpu.oracle_backward on the step's own rasterizer gradients (dL/dalpha_eff as its
    upstream dL/dalpha), camera included"""
    sc, _, dl, _, _ = _case()
    got = _step(sc, dl, aa=True, pose=True)
    du, dc, da, dcol, _ = got["raster"]
    N = len(sc["pws"])
    up = (du.reshape(N, 2), dc.reshape(N, 3), dcol.reshape(N, 3), np.zeros(N), da.reshape(N))
    ref, st, s, _ = oracle_backward(sc, K3, up)
    for k in ("pws", "shs", "scales", "rots", "alphas"):
        _eq(got["grads"][k], ref[k], k)
    _eq(got["per"], ref["cam"], "camera")
    # the frame is the colour oracle's on alpha_eff = rho alpha
    fwd = orc.splat(H, W, st["us"], st["ci"], s["rho"] * sc["alphas"], st["depths"].copy(), st["col"],
                    st["areas"].copy())
    _eq(got["image"], fwd["image"], "image")
    assert (s["rho"][st["keep"]] < 0.5).any()


def test_rgbd_alone_is_chain_plus_chain_depth(serial):
    sc, _, dl, dld, dla = _case()
    got = _step(sc, dl, dld, dla, rgbd=True)
    st = opose.stages(sc["pws"], sc["rots"], sc["scales"], sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"],
                      sc["fy"], sc["cx"], sc["cy"], W, H)
    fwd = ordb.splat_rgbd(H, W, st["us"], st["ci"], sc["alphas"], st["depths"].copy(), st["col"], st["areas"].copy())
    for k in ("image", "depth", "alpha"):
        _eq(got[k], fwd[k], k)
    du, dc, da, dcol, dz = ordb.splat_backward_rgbd(H, W, st["us"], st["ci"], sc["alphas"], st["col"], fwd["z"], fwd,
                                                    dl, dld, dla)
    ref = orc.chain_backward(sc["Rcw"], du, dc, da, dcol, *st["J"])
    _eq(got["grads"]["pws"], ref["pws"] + ordb.chain_depth(sc["Rcw"], dz, st["depths"]), "pws")
    for k in ("shs", "scales", "rots", "alphas", "us"):
        _eq(got["grads"][k], ref[k], k)
    assert np.abs(dz).max() > 0


def test_pose_alone_is_camera_grad(serial):
    sc, _, dl, _, _ = _case()
    got = _step(sc, dl, pose=True)
    base = _step(sc, dl)
    for k in base["grads"]:
        _eq(got["grads"][k], base["grads"][k], k)
    du, dc, da, dcol, _ = got["raster"]
    ref = opose.camera_grad(got["fwd"]["st"], sc["pws"], sc["Rcw"], sc["fx"], sc["fy"], W, H, du, dc, dcol)
    _eq(got["per"], ref["per"], "per")
    _eq(got["cam_grad"], ref["grad"], "grad")
    _eq(got["absum"], ref["absum"], "absum")


def test_filter_alone_is_chain_then_filter_backward(serial):
    """the colour chain on s', alpha' taken back through filter3d_oracle.backward
    (test_filter3d_cpu.test_oracle_chain_vs_central_differences's composition)"""
    sc, _, dl, _, _ = _case()
    f = _filter(sc)
    assert (f > 0).all()
    got = _step(sc, dl, filt=f)
    sf, af, _ = of3.apply(sc["scales"], sc["alphas"], f)
    st = opose.stages(sc["pws"], sc["rots"], sf, sc["shs"], sc["Rcw"], sc["tcw"], sc["twc"], sc["fx"], sc["fy"],
                      sc["cx"], sc["cy"], W, H)
    fwd = orc.splat(H, W, st["us"], st["ci"], af, st["depths"].copy(), st["col"], st["areas"].copy())
    g4 = orc.splat_backward(H, W, st["us"], st["ci"], af, st["col"], fwd, dl)
    ch = orc.chain_backward(sc["Rcw"], *g4, *st["J"])
    gs, ga = of3.backward(sc["scales"], sc["alphas"], f, ch["scales"], np.asarray(g4[2]).reshape(-1))
    _eq(got["image"], fwd["image"], "image")
    _eq(got["grads"]["scales"], gs, "scales")
    _eq(got["grads"]["alphas"], ga, "alphas")
    for k in ("pws", "shs", "rots", "us"):
        _eq(got["grads"][k], ch[k], k)


# ---------------------------------------------------------------- every flag on: central differences
def test_all_flags_vs_central_differences():
    """RGB-D + pose + AA + filter on a 300-Gaussian SH degree 3 scene with a general pose: about 80
    sampled parameters (65 of unflagged Gaussians the rasterizer used, all 15 camera entries) against
    central differences of the composed forward.  The forward is only piecewise smooth (threshold flips):
    test_filter3d_cpu's three step sizes, a parameter passes when one of them reproduces the analytic
    value, and 85 % of them must (at most 2 of the 15 camera entries may fail)."""
    k3 = 16
    sc = _scene(300, k3, seed=41)
    N = len(sc["pws"])
    rng = np.random.default_rng(42)
    sc["alphas"] = rng.uniform(0.05, 1.0, N).astype(np.float32)
    sc["scales"] = (sc["scales"] * rng.uniform(0.1, 1.0, (N, 1))).astype(np.float32)  # sub-pixel rows: AA, filter
    f = _filter(sc, seed=43)
    dl = upstream_gradient(W, H, 44) * np.float32(3.0 * W * H)
    dld = (rng.normal(size=(H, W)) * 0.3).astype(np.float32)
    dla = rng.normal(size=(H, W)).astype(np.float32)
    cam = ost.camera(sc, W, H)
    cam.update({k: np.array(sc[k], np.float32) for k in ("Rcw", "tcw", "twc")})
    flags = dict(rgbd=True, pose=True, aa=True, filt=f)
    ref = ost.step(sc, cam, dl=dl, dld=dld, dla=dla, **flags)
    rho = ref["fwd"]["rho"]
    assert (f > 0).all() and (rho[ref["fwd"]["st"]["keep"]] < 0.5).any()
    L0 = ost.loss(ost.render(cam, True, _own_inputs(sc, cam, f)), dl, dld, dla)

    def L(scene, c):
        return ost.loss(ost.render(c, True, _own_inputs(scene, c, f)), dl, dld, dla)

    drawn = np.zeros(N, bool)
    drawn[np.unique(_gsid(sc, cam, f))] = True
    pick = np.flatnonzero(drawn & ~ref["flagged"])
    assert len(pick) > 100
    params = []
    for _ in range(65):
        i = int(rng.choice(pick))
        name = str(rng.choice(["pws", "shs", "scales", "rots", "alphas"], p=[0.25, 0.2, 0.25, 0.15, 0.15]))
        j = 0 if name == "alphas" else int(rng.integers(sc[name].shape[1]))
        params.append((name, i, j))
    params += [("cam", c, 0) for c in range(15)]
    good, bad = 0, []
    for name, i, j in params:
        if name == "cam":
            key, idx = ("Rcw", divmod(i, 3)) if i < 9 else (("tcw", i - 9) if i < 12 else ("twc", i - 12))
            arr = cam[key]
            an = float(ref["cam_grad"][i])
        else:
            key, idx = name, ((i, j) if name != "alphas" else i)
            arr = sc[key]
            an = float(ref["grads"][name][i] if name == "alphas" else ref["grads"][name][i, j])
        x0 = float(arr[idx])
        ok = False
        for rel in (2e-3, 5e-4, 1.5e-4):
            h = rel * max(abs(x0), 0.05 if name == "alphas" else 1e-3)
            xp, xm = np.float32(x0 + h), np.float32(x0 - h)
            vals = []
            for x in (xp, xm):
                arr[idx] = x
                vals.append(L(sc, cam))
            arr[idx] = np.float32(x0)
            fd = (vals[0] - vals[1]) / (float(xp) - float(xm))
            # (a camera entry sums every drawn Gaussian's contribution, so a threshold flip anywhere in
            # the frame moves its quotient: ~1 % of absum, measured; the AA and depth camera addends are
            # under 0.5 % of absum here and are pinned by the exactness tests above instead)
            floor = 1e-2 * ref["absum"][i] if name == "cam" else 1e-6 * abs(L0)
            if abs(fd - an) <= 1e-2 * max(abs(fd), abs(an)) + floor:
                ok = True
                break
        good += ok
        if not ok:
            bad.append((name, i, j, an, fd))
    assert good >= int(0.85 * len(params)), "only %d of %d agree; %r" % (good, len(params), bad[:8])
    cam_bad = [b for b in bad if b[0] == "cam"]
    assert len(cam_bad) <= 2, cam_bad


def _own_inputs(scene, cam, f):
    fw = ost.forward(scene, cam, aa=True, filt=f)
    st = fw["st"]
    return dict(us=st["us"], ci=st["ci"], col=st["col"], depths=st["depths"], areas=st["areas"], alphas=fw["drawn"])


def _gsid(scene, cam, f):
    return ost.render(cam, True, _own_inputs(scene, cam, f))["gsid"]
