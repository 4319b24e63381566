"""Multi-GPU gradient exchange (SURVEY 8e; csrc/comm.cu + the PUSH variant of the fused
backward): `world` ranks are SIMULATED in one process on one GPU -- every rank has its own
region (gsb_comm_alloc), its own stream, its own camera and upstream gradients -- so the whole
protocol (tile ownership, peer stores, arrival / done flags, epoch re-arming, padding rows) runs
in the ordinary 1-GPU test suite.  The result must equal the rank-ordered sum of what the
single-GPU backward (ops.preprocessB) returns for each rank (to 1e-6 of the largest gradient:
the two kernel instantiations may differ by an ulp; dL/dalpha exactly).  The CUDA-IPC mapping
between real processes is exercised by bench.py --gpus N (benchmarks/gpu_extra.sh mgpu)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.mark.parametrize("world,N,k3", [(1, 1000, 16), (2, 1000, 16), (4, 5000, 4), (8, 70001, 16), (2, 128, 1)])
def test_exchange_equals_rank_ordered_sum(world, N, k3):
    from easygaussiansplatting_b200 import ops
    from easygaussiansplatting_b200.gsfunction import Camera
    from easygaussiansplatting_b200.parallel import GradExchange, rows_per_rank
    from easygaussiansplatting_b200.scene import ring_camera, synthetic_scene
    W, H = 320, 200
    sc = synthetic_scene(N, W, H, sh_dim=3 * k3, seed=world)
    pws, rots, scales, shs = t(sc["pws"]), t(sc["rots"] * 1.3), t(sc["scales"]), t(sc["shs"])
    nbytes = GradExchange.region_bytes(N, k3, world)
    assert nbytes >= 4096 + 2 * world * rows_per_rank(N, world) * (3 * k3 + 11) * 4
    regions = [GradExchange.alloc_region(nbytes)[0] for _ in range(world)]
    exs = [GradExchange(N, k3, world, r, regions, DEV, own_region=regions[r]) for r in range(world)]
    streams = [torch.cuda.Stream() for _ in range(world)]
    try:
        for step in range(3):
            g = torch.Generator(device=DEV).manual_seed(100 * world + step)
            cams, ins, local = [], [], []
            for r in range(world):
                Rcw, tcw, twc = ring_camera(r + step, world + 2)
                cams.append(Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(Rcw), t(tcw), t(twc)))
                ins.append([torch.randn((N, 1, k), device=DEV, generator=g) for k in (2, 3, 3, 1)])  # us cinv colors alpha
                gu, gc, gcol, ga = ins[-1]
                dpws, dshs, dscales, drots = ops.preprocessB(pws, rots, scales, shs, cams[r].Rcw, cams[r].tcw,
                                                            cams[r].twc, sc["fx"], sc["fy"], sc["cx"], sc["cy"], W, H,
                                                            gu, gc, gcol)
                local.append(dict(dpws=dpws, dshs=dshs, dscales=dscales, drots=drots, dalphas=ga.reshape(N, 1)))
            want = {k: local[0][k].clone() for k in local[0]}
            for r in range(1, world):
                for k in want:
                    want[k] += local[r][k]
            torch.cuda.synchronize()
            for r in range(world):
                with torch.cuda.stream(streams[r]):
                    exs[r].push(pws, rots, scales, shs, cams[r], *ins[r])
            if step == 0:
                torch.cuda.synchronize()          # first step: phases separated; later steps overlap freely
            outs = []
            for r in range(world):
                with torch.cuda.stream(streams[r]):
                    outs.append(exs[r].reduce())
            torch.cuda.synchronize()
            for r in range(world):
                assert exs[r].status() == 0, "rank %d: a flag wait timed out" % r
                for k in want:
                    assert outs[r][k].shape == want[k].shape
                    # the PUSH and local instantiations of the backward kernel are compiled
                    # separately; ptxas may contract a*b+c*d differently (seen: 1 ulp at k3 = 1)
                    err = float((outs[r][k] - want[k]).abs().max() / want[k].abs().max().clamp_min(1e-30))
                    assert err <= 5e-6, (step, r, k, err)
                    if k == "dalphas":
                        assert torch.equal(outs[r][k], want[k])      # pure pass-through + rank-ordered sum
    finally:
        for ex in exs:
            ex.close()


def test_exchange_through_autograd_single_rank():
    """GSFunctionFused with cam.grad_exchange set (world 1) returns the same gradients as without"""
    from easygaussiansplatting_b200.gsfunction import Camera, GSFunctionFused
    from easygaussiansplatting_b200.parallel import GradExchange
    from easygaussiansplatting_b200.scene import synthetic_scene, upstream_gradient
    N, W, H = 3000, 256, 160
    sc = synthetic_scene(N, W, H, sh_dim=48, seed=4)
    cam = Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(sc["Rcw"]), t(sc["tcw"]), t(sc["twc"]))
    dl = t(upstream_gradient(W, H, 4) * (3.0 * W * H))
    region, _ = GradExchange.alloc_region(GradExchange.region_bytes(N, 16, 1))
    ex = GradExchange(N, 16, 1, 0, [region], DEV, own_region=region)
    got = {}
    try:
        for mode in ("plain", "exchange"):
            leaves = [t(sc[k]).requires_grad_() for k in ("pws", "shs")] + [t(sc["alphas"][:, None]).requires_grad_()] + \
                     [t(sc[k]).requires_grad_() for k in ("scales", "rots")]
            us = torch.zeros((N, 2), device=DEV, requires_grad=True)
            cam.grad_exchange = ex if mode == "exchange" else None
            img, _ = GSFunctionFused.apply(leaves[0], leaves[1], leaves[2], leaves[3], leaves[4], us, cam)
            img.backward(dl)
            got[mode] = [p.grad.clone() for p in leaves] + [us.grad.clone()]
        assert ex.status() == 0
        for a, b in zip(got["plain"], got["exchange"]):
            assert float((a - b).abs().max() / a.abs().max().clamp_min(1e-30)) <= 1e-6
    finally:
        ex.close()


def test_exchange_argument_errors():
    from easygaussiansplatting_b200 import _lib
    lib = _lib.load()
    assert lib.gsb_exchange_region_bytes(1000, 16, 9) == 0
    assert lib.gsb_exchange_region_bytes(1000, 16, 2) > 0
    import ctypes as C
    regs = (C.c_void_p * 2)(None, None)
    rc = lib.gsb_grad_reduce_broadcast(1000, 16, 2, 0, regs, 1, None)
    assert rc != 0 and b"null region" in lib.gsb_last_error()
    rc = lib.gsb_grad_reduce_broadcast(1000, 16, 2, 0, regs, 0, None)
    assert rc != 0
    # push checks the parameter set like preprocessB: rots / scales with N - 1 rows or a short
    # camera tensor raise before any launch (the kernel reads N rows and 9 / 3 floats)
    from easygaussiansplatting_b200.gsfunction import Camera
    from easygaussiansplatting_b200.parallel import GradExchange
    from easygaussiansplatting_b200.scene import synthetic_scene
    N, k3 = 1000, 16
    sc = synthetic_scene(N, 64, 64, sh_dim=3 * k3, seed=5)
    P = {k: t(sc[k]) for k in ("pws", "rots", "scales", "shs")}
    region, _ = GradExchange.alloc_region(GradExchange.region_bytes(N, k3, 1))
    ex = GradExchange(N, k3, 1, 0, [region], DEV, own_region=region)
    cam = dict(Rcw=t(sc["Rcw"]), tcw=t(sc["tcw"]), twc=t(sc["twc"]))
    ins = [torch.zeros((N, k), device=DEV) for k in (2, 3, 3, 1)]
    try:
        torch.cuda.synchronize()
        launches = lib.gsb_profile_launches(-1)
        for name, short in (("rots", P["rots"][:-1]), ("scales", P["scales"][:-1]),
                            ("Rcw", cam["Rcw"].reshape(-1)[:8]), ("tcw", cam["tcw"][:2]), ("twc", cam["twc"][:2])):
            p, c = dict(P), dict(cam)
            (p if name in p else c)[name] = short
            with pytest.raises(ValueError):
                ex.push(p["pws"], p["rots"], p["scales"], p["shs"],
                        Camera(64, 64, sc["fx"], sc["fy"], sc["cx"], sc["cy"], c["Rcw"], c["tcw"], c["twc"]), *ins)
        # so are the upstream gradients: a dloss_dcinv2ds or dloss_dcolors with N - 1 rows (3N floats read)
        for i in (1, 2):
            short = list(ins)
            short[i] = ins[i][:-1]
            with pytest.raises(ValueError):
                ex.push(P["pws"], P["rots"], P["scales"], P["shs"],
                        Camera(64, 64, sc["fx"], sc["fy"], sc["cx"], sc["cy"], cam["Rcw"], cam["tcw"], cam["twc"]),
                        *short)
        assert lib.gsb_profile_launches(-1) == launches
    finally:
        ex.close()


@pytest.mark.parametrize("world,N,k3", [(2, 3001, 1), (4, 3001, 9), (2, 20001, 9), (4, 20001, 1)])
def test_exchange_with_moment_rows_equals_rank_ordered_sum(world, N, k3):
    """push(moments=..., cinv2ds=...) -- the k_preprocess_bwd<K3, PUSH, MOM> kernel training runs
    across GPUs -- against the rank-ordered sum of each rank's local preprocessB(moments=...), at
    odd N (ragged last tile, padding rows in the slots); this rank's dL/du comes back unsummed."""
    from easygaussiansplatting_b200 import ops
    from easygaussiansplatting_b200.gsfunction import Camera
    from easygaussiansplatting_b200.parallel import GradExchange
    from easygaussiansplatting_b200.scene import ring_camera, synthetic_scene
    W, H = 320, 200
    sc = synthetic_scene(N, W, H, sh_dim=3 * k3, seed=world + 10)
    pws, rots, scales, shs = t(sc["pws"]), t(sc["rots"] * 1.3), t(sc["scales"]), t(sc["shs"])
    regions = [GradExchange.alloc_region(GradExchange.region_bytes(N, k3, world))[0] for _ in range(world)]
    exs = [GradExchange(N, k3, world, r, regions, DEV, own_region=regions[r]) for r in range(world)]
    streams = [torch.cuda.Stream() for _ in range(world)]
    names = ("dpws", "dshs", "dscales", "drots", "dus", "dalphas")
    try:
        for step in range(3):
            g = torch.Generator(device=DEV).manual_seed(1000 * world + step)
            cams, ins, local = [], [], []
            for r in range(world):
                Rcw, tcw, twc = ring_camera(r + step, world + 2)
                cams.append(Camera(W, H, sc["fx"], sc["fy"], sc["cx"], sc["cy"], t(Rcw), t(tcw), t(twc)))
                cinv2ds = ops.preprocess(pws, rots, scales, shs, cams[r].Rcw, cams[r].tcw, cams[r].twc, sc["fx"],
                                         sc["fy"], sc["cx"], sc["cy"], W, H)[1]
                moments = torch.randn((N, 9), device=DEV, generator=g)
                moments[torch.rand(N, device=DEV, generator=g) < 0.05, 0:2] = 0   # untouched rows
                ins.append((moments, cinv2ds))
                out = ops.preprocessB(pws, rots, scales, shs, cams[r].Rcw, cams[r].tcw, cams[r].twc, sc["fx"],
                                      sc["fy"], sc["cx"], sc["cy"], W, H, None, None, None, moments=moments,
                                      cinv2ds=cinv2ds)
                local.append(dict(zip(names, out)))
                local[-1]["dalphas"] = local[-1]["dalphas"].reshape(N, 1)
            want = {k: local[0][k].clone() for k in names if k != "dus"}
            for r in range(1, world):
                for k in want:
                    want[k] += local[r][k]
            torch.cuda.synchronize()
            dus = []
            for r in range(world):
                with torch.cuda.stream(streams[r]):
                    dus.append(exs[r].push(pws, rots, scales, shs, cams[r], moments=ins[r][0], cinv2ds=ins[r][1]))
            outs = []
            for r in range(world):
                with torch.cuda.stream(streams[r]):
                    outs.append(exs[r].reduce())
            torch.cuda.synchronize()
            for r in range(world):
                assert exs[r].status() == 0, "rank %d: a flag wait timed out" % r
                assert torch.equal(dus[r], local[r]["dus"]), (step, r)
                for k in want:
                    assert outs[r][k].shape == want[k].shape
                    err = float((outs[r][k] - want[k]).abs().max() / want[k].abs().max().clamp_min(1e-30))
                    assert err <= 5e-6, (step, r, k, err)
                assert torch.equal(outs[r]["dalphas"], want["dalphas"]), (step, r)
    finally:
        for ex in exs:
            ex.close()
