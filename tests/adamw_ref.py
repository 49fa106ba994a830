"""Float64 reference of one step of rb_clip_adamw / rb_peer_adamw_gather (clip + AdamW with Adam state per parameter group)
in torch semantics, built on tests/adam_ref.py and its scale conventions:
  torch.nn.utils.clip_grad_norm_ over ALL groups: one global norm, coef = min(max_norm / (norm + 1e-6), 1);
  torch.optim.AdamW per group g (lambda_g, t_g = group_steps[g] + 1):
      p_d = p (1 - lr lambda_g)                 (param.mul_(1 - lr * weight_decay), before the moments)
      then adam_ref's Adam step from p_d with the bias corrections of t_g.
Scales: m' and v' as adam_ref; p' as adam_ref with |p| replaced by |p| + |p| lr lambda_g (the decay's product carries the
scale of p).  TAU is adam_ref.TAU; tests/test_adamw_host.py checks it against an fp32 model of the kernel and against the
slips it must catch."""
import torch

import adam_ref as AR

TAU = AR.TAU


def clip_adamw(p, g, m, v, groups, group_steps, grad_scale, max_norm, lr, b1, b2, eps):
    """One step from fp32 tensors.  groups: [(begin, end, weight_decay)] tiling [0, P); group_steps: each group's count
    before the step.  Returns adam_ref.clip_adam's dict (p, m, v as (value, scale) over all P elements, norm, coef)."""
    f = lambda x: float(torch.tensor(x, dtype=torch.float32))      # the kernel's fp32 arguments
    lr32 = f(lr)
    gs = g.double() * f(grad_scale)
    norm = float(gs.square().sum().sqrt())
    coef = min(f(max_norm) / (norm + 1e-6), 1.0)
    out = {k: (torch.empty(p.numel(), dtype=torch.float64, device=p.device),
               torch.empty(p.numel(), dtype=torch.float64, device=p.device)) for k in ("p", "m", "v")}
    for (b, e, wd), t in zip(groups, group_steps):
        keep = 1.0 - lr32 * f(wd)
        pd = p[b:e].double() * keep
        # the group's step with the global clip coefficient: adam_ref with max_norm = inf and the gradient pre-clipped
        r = AR.clip_adam(pd, (gs[b:e] * coef), m[b:e], v[b:e], t, 1.0, float("inf"), lr32, b1, b2, eps)
        for k in ("m", "v"):
            out[k][0][b:e], out[k][1][b:e] = r[k]
        out["p"][0][b:e] = r["p"][0]
        out["p"][1][b:e] = r["p"][1] + p[b:e].double().abs() * lr32 * f(wd)
    return dict(p=out["p"], m=out["m"], v=out["v"], norm=(norm, norm + AR.FLOOR), coef=coef)
