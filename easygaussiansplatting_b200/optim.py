"""GaussianAdam: torch.optim.Adam's step as one sm_90a kernel launch (gsb_adam_step, DESIGN 3.12),
with an optional visibility mask (selective Adam).

    optimizer = GaussianAdam(adam_params, eps=1e-15)       # in place of torch.optim.Adam
    ...
    image, mask = GSFunctionFused.apply(...)               # mask: depths > 0.2, [N] bool
    loss.backward()
    optimizer.step(visibility=mask)                        # or step() for dense Adam

Dense steps follow torch's foreach Adam (the default for CUDA params) operation for operation in
fp32.  The state layout is torch.optim.Adam's (`step` a CPU float32 scalar, `exp_avg` and
`exp_avg_sq` shaped like the param, created on the first step that sees a grad) and so are the
param-group keys, so state_dict() / load_state_dict() carry over in both directions, and
DensityController / MCMCController work on either optimizer.
"""
import ctypes as C

import torch

from . import _lib


class GaussianAdam(torch.optim.Optimizer):
    """Adam over fp32, contiguous CUDA params, one kernel launch per step.

    step(visibility=None) is dense Adam.  step(visibility=mask) with a bool / uint8 CUDA tensor
    [N] is selective Adam (gsplat's SelectiveAdam): every param with a grad must be [N, D]; rows
    whose mask is 0 keep their param and both moments exactly, and their grad is not read.  The
    step count is per tensor and advances on every call that sees a grad, whatever the mask.
    Params whose grad is None are skipped and their step does not advance.  amsgrad, weight_decay,
    maximize and capturable are refused.  step() does not synchronise with the device."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, *,
                 foreach=None, maximize=False, capturable=False, differentiable=False, fused=None,
                 decoupled_weight_decay=False):
        if not 0.0 <= lr:
            raise ValueError("Invalid learning rate: %r" % (lr,))
        if not 0.0 <= eps:
            raise ValueError("Invalid epsilon value: %r" % (eps,))
        if not (0.0 <= betas[0] < 1.0 and 0.0 <= betas[1] < 1.0):
            raise ValueError("Invalid beta parameters: %r" % (betas,))
        # torch.optim.Adam's keys, so that its state_dict loads here and ours loads there
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad, maximize=maximize,
                        foreach=foreach, capturable=capturable, differentiable=differentiable, fused=fused,
                        decoupled_weight_decay=decoupled_weight_decay)
        super().__init__(params, defaults)
        for group in self.param_groups:
            self._check_group(group)

    @staticmethod
    def _check_group(group):
        for key in ("amsgrad", "maximize", "capturable", "differentiable"):
            if group.get(key, False):
                raise ValueError("GaussianAdam does not support %s=True" % key)
        if group.get("weight_decay", 0) != 0:
            raise ValueError("GaussianAdam does not support weight_decay")
        for p in group["params"]:
            if not p.is_cuda or p.dtype != torch.float32:
                raise ValueError("GaussianAdam takes float32 CUDA params (there is no CPU fallback), got %s on %s"
                                 % (p.dtype, p.device))
            if not p.is_contiguous():
                raise ValueError("GaussianAdam params must be contiguous")

    def add_param_group(self, param_group):
        super().add_param_group(param_group)
        self._check_group(self.param_groups[-1])

    @staticmethod
    def _moment(st, key, p):
        t = st[key]
        if t.shape != p.shape or t.dtype != torch.float32 or t.device != p.device or not t.is_contiguous():
            raise ValueError("state[%r] must be a contiguous float32 tensor shaped and placed like its param" % key)
        return t

    @torch.no_grad()
    def step(self, closure=None, visibility=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        N = 0
        vis = None
        if visibility is not None:
            if not isinstance(visibility, torch.Tensor) or visibility.dtype not in (torch.bool, torch.uint8) \
                    or visibility.dim() != 1 or not visibility.is_cuda:
                raise ValueError("visibility must be a 1-D bool or uint8 CUDA tensor [N]")
            vis = visibility.contiguous()
            N = vis.shape[0]
        # one launch per (beta1, beta2, eps); the usual single setting gives one launch per step
        batches = {}
        keep = []
        for group in self.param_groups:
            self._check_group(group)
            beta1, beta2 = (float(b) for b in group["betas"])
            lr = float(group["lr"])
            for p in group["params"]:
                if p.grad is None:
                    continue
                g = p.grad
                if g.is_sparse:
                    raise ValueError("GaussianAdam does not support sparse gradients")
                if g.shape != p.shape or g.dtype != torch.float32 or g.device != p.device:
                    raise ValueError("a grad must be float32 and shaped and placed like its param")
                if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous():
                    raise ValueError("GaussianAdam takes contiguous float32 CUDA params")
                if vis is not None and (p.dim() != 2 or p.shape[0] != N or p.device != vis.device):
                    raise ValueError("selective steps take [N, D] params with N = %d (the visibility's length), "
                                     "got %s" % (N, tuple(p.shape)))
                g = g.contiguous()
                st = self.state[p]
                if len(st) == 0:
                    st["step"] = torch.tensor(0.0, dtype=torch.float32)
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                m, v = self._moment(st, "exp_avg", p), self._moment(st, "exp_avg_sq", p)
                st["step"] += 1
                t = float(st["step"].item())  # a CPU scalar: no device synchronisation
                # torch.optim.adam._multi_tensor_adam's bias corrections, in double
                step_size = lr / (1 - beta1 ** t)
                bc2_sqrt = (1 - beta2 ** t) ** 0.5
                keep.append(g)
                row = _lib.AdamTensor(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(),
                                      p.shape[1] if vis is not None else 0, step_size, bc2_sqrt)
                batches.setdefault((beta1, beta2, float(group["eps"])), []).append(row)
        if batches:
            lib = _lib.load()
            stream = C.c_void_p(torch.cuda.current_stream(vis.device if vis is not None else None).cuda_stream)
            for (beta1, beta2, eps), rows in batches.items():
                table = (_lib.AdamTensor * len(rows))(*rows)
                _lib.check(lib.gsb_adam_step(len(rows), table, N, C.c_void_p(vis.data_ptr() if vis is not None else 0),
                                             beta1, beta2, eps, stream), lib)
        return loss
