"""CPU oracle for the fused Adam step (DESIGN 3.12).  TEST INFRASTRUCTURE ONLY -- imported by tests/
(and nothing in the product).

Adam in fp64 on fp32 (or fp64) inputs, the textbook form torch.optim.Adam implements:
    m = beta1 m + (1 - beta1) g,  v = beta2 v + (1 - beta2) g^2,
    p = p - lr / (1 - beta1^t) * m / (sqrt(v) / sqrt(1 - beta2^t) + eps)
with t the tensor's step count after the increment.  Selective Adam updates only the rows whose
visibility is set and leaves the others' p, m and v as they were; the step count still advances
on every call (gsplat's SelectiveAdam).
"""
import numpy as np


def adam_update(p, g, m, v, t, lr, beta1=0.9, beta2=0.999, eps=1e-8):
    """one Adam update at step count t (>= 1) -> (p, m, v) in fp64"""
    p, g, m, v = (np.asarray(x, np.float64) for x in (p, g, m, v))
    m = beta1 * m + (1.0 - beta1) * g
    v = beta2 * v + (1.0 - beta2) * g * g
    denom = np.sqrt(v) / np.sqrt(1.0 - beta2 ** t) + eps
    p = p - lr / (1.0 - beta1 ** t) * m / denom
    return p, m, v


def adam_step(p, g, m, v, t, lr, beta1=0.9, beta2=0.999, eps=1e-8, visibility=None):
    """one step of dense (visibility None) or selective Adam on one [N, ...] tensor whose step count
    was t before the call -> (p, m, v, t + 1), fp64; invisible rows are the inputs unchanged"""
    t = t + 1
    pn, mn, vn = adam_update(p, g, m, v, t, lr, beta1, beta2, eps)
    if visibility is not None:
        keep = ~np.asarray(visibility, bool)
        for new, old in ((pn, p), (mn, m), (vn, v)):
            new[keep] = np.asarray(old, np.float64)[keep]
    return pn, mn, vn, t
