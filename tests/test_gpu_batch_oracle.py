"""The batched step (GSFunctionFusedBatch[RGBD], DESIGN 3.21) against the fp64 whole-step oracle: the sum
over the cameras of oracle.step_oracle.step(scene, cam_c, ...) on test_gpu_step_matrix's edge-row scene
(culled, fov-clamped, zero-scale, needle and huge rows, filter edge rows), three cameras with their own
poses and intrinsics, with and without antialiasing and the 3D filter, colour and RGB-D, at that file's
bounds.  This holds k_preprocess_bwd_batch's register sum over the cameras, and the batch rasterizers, to
an independent reference rather than to the single-camera path."""
import numpy as np
import pytest
import torch

from oracle import step_oracle as ost
from easygaussiansplatting_b200.scene import ring_camera

from test_gpu_step_matrix import (GRADS, N_MAT, _camera, _upstream, bits, check_grads, check_planes, drawn_frame,
                                  matrix_scene, n, t)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("filt", [False, True])
@pytest.mark.parametrize("aa", [False, True])
def test_batch_step_vs_oracle(aa, filt):
    from easygaussiansplatting_b200.gsfunction import GSFunctionFusedBatch, GSFunctionFusedBatchRGBD
    W, H, k3, C = 640, 360, 16, 3
    rgbd = aa != filt  # both frame families over the four cases
    sc, f, rows = matrix_scene(N_MAT, W, H, k3, seed=401 + 2 * aa + 4 * filt)
    f = f if filt else None
    vscs, cams = [], []
    for v in range(C):
        R, tc, tw = ring_camera(v, 8)
        vsc = dict(sc, Rcw=R, tcw=tc, twc=tw, fx=sc["fx"] * (1.0 + 0.05 * v), fy=sc["fy"] * (1.0 + 0.03 * v),
                   cx=sc["cx"] + 3.0 * v, cy=sc["cy"] - 2.0 * v)
        vscs.append(vsc)
        cams.append(_camera(vsc, W, H, aa))
    ups = [_upstream(W, H, 20 + v) for v in range(C)]
    P = {k: t(sc[k]).requires_grad_() for k in ("pws", "shs", "scales", "rots")}
    al = t(sc["alphas"][:, None]).requires_grad_()
    us = torch.zeros((C, N_MAT, 2), device=DEV, requires_grad=True)
    F = GSFunctionFusedBatchRGBD if rgbd else GSFunctionFusedBatch
    outs = F.apply(P["pws"], P["shs"], al, P["scales"], P["rots"], us, cams, None if f is None else t(f))
    loss = 0.0
    for v, (dl, dld, dla) in enumerate(ups):
        loss = loss + (outs[0][v] * t(dl)).sum()
        if rgbd:
            loss = loss + (outs[1][v] * t(dld)).sum() + (outs[2][v] * t(dla)).sum()
    loss.backward()
    views = []
    for v, (vsc, cam, (dl, dld, dla)) in enumerate(zip(vscs, cams, ups)):
        inp, ref = drawn_frame(vsc, cam, f, rgbd)
        assert torch.equal(bits(outs[0][v]), bits(ref[0]))
        if rgbd:
            assert torch.equal(bits(outs[1][v]), bits(ref[5])) and torch.equal(bits(outs[2][v]), bits(ref[6]))
        o = ost.step(vsc, ost.camera(vsc, W, H), rgbd=rgbd, pose=False, aa=aa, filt=f, dl=dl,
                     dld=dld if rgbd else None, dla=dla if rgbd else None, drawn_inputs=inp)
        check_planes([x[v] for x in outs[:3 if rgbd else 1]], o, rgbd)
        views.append(o)
    got = dict(pws=n(P["pws"].grad), shs=n(P["shs"].grad), scales=n(P["scales"].grad), rots=n(P["rots"].grad),
               alphas=n(al.grad))
    want = {k: sum(o["grads"][k] for o in views) for k in GRADS if k != "us"}
    flagged = np.any([o["flagged"] for o in views], axis=0)
    band = np.any([o["band"] for o in views], axis=0)
    thin = np.any([o["thin"] for o in views], axis=0)
    check_grads(got, want, flagged, band, thin, names=tuple(want))
    for v, o in enumerate(views):
        check_grads({"us": n(us.grad[v])}, o["grads"], o["flagged"], o["band"], o["thin"], names=("us",))
    if filt:  # rows never composited in any view: no gradient at all
        dead = np.concatenate([rows["f_huge"], rows["zero_axis"]])
        for k in want:
            assert not got[k].reshape(N_MAT, -1)[dead].any(), k
