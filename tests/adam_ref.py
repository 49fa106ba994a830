"""Float64 reference of one optimiser step of rb_clip_adam (csrc/rb_kernels.cu k_sqnorm + k_clip_adam) in torch semantics,
with a condition scale for every output element:
  torch.nn.utils.clip_grad_norm_   norm = ||g s||, coef = min(max_norm / (norm + 1e-6), 1), g' = g s coef;
  torch.optim.Adam (no amsgrad, no weight decay), t = step_count + 1:
                                   m' = m + (g' - m)(1 - b1)             (exp_avg.lerp_)
                                   v' = v b2 + (1 - b2) g'^2
                                   p' = p - lr / (1 - b1^t) * m' / (sqrt(v') / sqrt(1 - b2^t) + eps).
Computed from the same fp32 tensors the kernel reads (its own state before the step).  Scales, in the spirit of
tests/head_ref.py (sum of the absolute values of the terms that make the element):
  norm  norm;   m'  |m| + |g'|;   v'  |v| b2 + (1 - b2) g'^2;
  p'    |p| + step_size (|m| + |g'|) / denom, the update carrying the scale of m' (the kernel's m' feeds it) and the
        relative error of sqrt.approx.f32 / rcp.approx.f32 (both within 2^-23 relative, PTX ISA) of the denominator.
Every scale carries FLOOR = FLT_MIN: below fp32's normal range the spacing is absolute (2^-149), and TAU * FLT_MIN is
16 of those, so tiny gradients whose v' is subnormal are held to what fp32 can represent there.
TAU is derived in tests/test_c51_adam_bounds.py: at least 5x above the fp32 arithmetic (the CPU oracle and a model of
the kernel's operations with the approximate sqrt / reciprocal perturbed by their stated bounds), at least 5x below each
semantic slip it tests."""
import math

import torch

TAU = 2e-6
FLOOR = 2.0 ** -126


def clip_adam(p, g, m, v, step_count, grad_scale, max_norm, lr, b1, b2, eps):
    """One step from fp32 tensors (any device).  step_count: the kernel's count before the step.  Returns
    dict(p=(p', scale), m=(..), v=(..), norm=(norm, scale), coef=coef) in float64."""
    f = lambda x: float(torch.tensor(x, dtype=torch.float32))          # the kernel's fp32 arguments
    grad_scale, max_norm, lr, b1, b2, eps = (f(x) for x in (grad_scale, max_norm, lr, b1, b2, eps))
    p, g, m, v = (t.double() for t in (p, g, m, v))
    gs = g * grad_scale
    norm = float(gs.square().sum().sqrt())
    coef = min(max_norm / (norm + 1e-6), 1.0)
    gc = gs * coef
    m1 = m + (gc - m) * (1 - b1)
    v1 = v * b2 + (1 - b2) * gc.square()
    t = step_count + 1
    bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
    step_size = lr / bc1
    denom = v1.sqrt() / math.sqrt(bc2) + eps
    p1 = p - step_size * m1 / denom
    sm = m.abs() + gc.abs() + FLOOR
    return dict(p=(p1, p.abs() + step_size * sm / denom + FLOOR), m=(m1, sm), v=(v1, v.abs() * b2 + (1 - b2) * gc.square() + FLOOR),
                norm=(norm, norm + FLOOR), coef=coef)
