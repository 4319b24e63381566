"""The fused forward + backward captured in CUDA graphs (SURVEY 7 step 5: no host round trip, no
per-kernel launch cost).

Below ~500k Gaussians the step is bound by the host: ~25 launches and their Python wrappers per
step can cost more than the kernels themselves.  The capacity-based rasterizer, enqueue-only
(`ops._capacity_frame`), has no host decision inside the frame, so the whole forward (fused
per-Gaussian stage, binning, sort, rasterizer) and the whole backward replay as two graphs over
static buffers:

    step = GraphedFusedStep(pws, shs, alphas, scales, rots, cam)    # learns capacities, captures
    image = step.forward()                 # static tensor; camera = step.cam (update its tensors in place)
    step.dloss_dimage.copy_(...)           # the loss lives between the two graphs
    grads = step.backward()                # dict dpws dshs dalphas dscales drots dus (static tensors)

With cam.antialiased the captured frame composites alpha_eff = rho * alpha (ops.preprocess) and the
backward returns dL/dalpha of the raw alphas; binning, hence the captured capacities, is the same.
With filter3d[N] (ops.filter3d, the Mip-Splatting 3D filter) the forward graph starts with the
filter's apply pass (s', alpha') and the backward graph ends with its backward, so the gradients
are those of the unfiltered scales and alphas; the filter is captured by address like the
parameters (recompute it in place).

The parameters are captured by address: an optimizer that updates them in place is seen by the
next replay.  `forward()`'s outputs are validated lazily: `backward()` (or `check()`) reads the
binning status of the frame; a frame that outgrew the captured capacities raises `CapacityError`
after which `recapture()` (larger bounds) and a repeat of the step are due."""
import torch

from . import ops
from .gsfunction import camera_model_kwargs


class CapacityError(RuntimeError):
    pass


class GraphedFusedStep:
    def __init__(self, pws, shs, alphas, scales, rots, cam, headroom=1.5, filter3d=None):
        self.p = dict(pws=pws.detach(), shs=shs.detach(), alphas=alphas.detach(), scales=scales.detach(),
                      rots=rots.detach())
        self.filter3d = filter3d.detach() if filter3d is not None else None
        self.cam, self.headroom = cam, float(headroom)
        self.device = pws.device
        self.status = torch.zeros(4, dtype=torch.int32).pin_memory()
        self._done = torch.cuda.Event()
        self.recapture()

    # ------------------------------------------------------------------ capture
    def _drawn_params(self):
        """the scales and alphas the frame is rendered from: s', alpha' with the filter"""
        p = self.p
        if self.filter3d is None:
            return p["scales"], p["alphas"]
        return ops.filter3d_apply(p["scales"], p["alphas"], self.filter3d)

    def _learn_capacities(self):
        cam, p = self.cam, self.p
        scales, alphas = self._drawn_params()
        us, ci, col, dep, ar = ops.preprocess(p["pws"], p["rots"], scales, p["shs"], cam.Rcw, cam.tcw, cam.twc,
                                              cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height,
                                              **camera_model_kwargs(cam))
        out = ops.splat(cam.height, cam.width, us, ci, alphas, dep, col, ar)
        dkmax = int((dep.max().clamp_min(0) * 1000).item()) + 1
        return ops._next_capacity(out[4].numel(), dkmax, headroom=self.headroom)

    def _forward_body(self):
        cam, p = self.cam, self.p
        aa = bool(getattr(cam, "antialiased", False))
        scales, alphas = self._drawn_params()
        pre = ops.preprocess(p["pws"], p["rots"], scales, p["shs"], cam.Rcw, cam.tcw, cam.twc, cam.fx, cam.fy,
                             cam.cx, cam.cy, cam.width, cam.height, alphas=alphas, antialiased=aa,
                             **camera_model_kwargs(cam))
        us, ci, col, dep, ar, rec = pre[:6]
        drawn = pre[6] if aa else alphas  # antialiased: the rasterizers composite alpha_eff
        lib = ops._L()
        enqueue = (lib.gsb_splat_forward_enqueue, [ops._ptr(t) for t in (us, ci, drawn, dep, col, ar, rec)])
        _, self._keep, (image, contrib, final_tau, ranges, gsid) = ops._capacity_frame(
            cam.height, cam.width, us, [], lib.gsb_splat_workspace_bytes, enqueue, self.P_cap, self.dk_cap,
            self.status)
        self._fwd = dict(us=us, cinv2ds=ci, colors=col, depths=dep, areas=ar, records=rec, contrib=contrib,
                         final_tau=final_tau, ranges=ranges, gsid=gsid, alphas=drawn, aa=aa, scales_f=scales,
                         alphas_f=alphas)
        self.image = image

    def _backward_body(self):
        cam, p, f = self.cam, self.p, self._fwd
        # all P_cap patch slots: the replay's patch count is only known on the device
        moments = ops.splatB(cam.height, cam.width, f["us"], f["cinv2ds"], f["alphas"], f["depths"], f["colors"],
                             f["contrib"], f["final_tau"], f["ranges"], f["gsid"], self.dloss_dimage,
                             moments_only=True, records=f["records"])
        gpw, gsh, gs, gq, dus, dal = ops.preprocessB(
            p["pws"], p["rots"], f["scales_f"], p["shs"], cam.Rcw, cam.tcw, cam.twc, cam.fx, cam.fy, cam.cx, cam.cy,
            cam.width, cam.height, None, None, None, moments=moments, cinv2ds=f["cinv2ds"], antialiased=f["aa"],
            alphas=f["alphas_f"] if f["aa"] else None, **camera_model_kwargs(cam))
        if self.filter3d is not None:  # dL/ds', dL/dalpha' -> dL/ds, dL/dalpha, in place
            ops.filter3d_backward(p["scales"], p["alphas"], self.filter3d, gs, dal, inplace=True)
        self._keep_b = moments
        self.grads = dict(dpws=gpw, dshs=gsh, dscales=gs, drots=gq, dalphas=dal, dus=dus)

    def recapture(self, P_cap=None, dk_cap=None):
        """(re)learn the capacities from one exact frame and capture both graphs"""
        cam = self.cam
        with torch.cuda.device(self.device):
            learnt = self._learn_capacities()
            self.P_cap, self.dk_cap = int(P_cap or learnt[0]), int(dk_cap or learnt[1])
            self.dloss_dimage = torch.zeros((3, cam.height, cam.width), dtype=torch.float32, device=self.device)
            side = torch.cuda.Stream(device=self.device)
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):  # one eager pass on the capture stream: lazy initialisations
                self._forward_body()
                self._backward_body()
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            self.g_fwd, self.g_bwd = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.g_fwd):
                self._forward_body()
            with torch.cuda.graph(self.g_bwd, pool=self.g_fwd.pool()):
                self._backward_body()
        self._pending = False

    # ------------------------------------------------------------------ replay
    def forward(self):
        self.g_fwd.replay()
        self._done.record()
        self._pending = True
        return self.image

    def check(self):
        """waits for the last forward and validates its binning status -> the frame's patch count"""
        if self._pending:
            self._done.synchronize()
            self._pending = False
            P, _, flags = ops._decode_status(self.status)
            if (flags & (ops.GSB_STATUS_P_CAP | ops.GSB_STATUS_DEPTH_KEY)) or P > self.P_cap:
                raise CapacityError("frame outgrew the captured capacities (P = %d of %d, flags %d): "
                                    "recapture() and repeat the step" % (P, self.P_cap, flags))
        return ops._decode_status(self.status)[0]

    def backward(self):
        self.check()
        self.g_bwd.replay()
        return self.grads
