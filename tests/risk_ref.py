"""Float64 reference of the distorted values Q_beta of risk-sensitive selection (DESIGN.md §18; csrc/rb_kernels.cu:
c51_risk_value / qr_risk_value behind the six _risk entries), with a derived per-row error bound, and an fp32 emulation
of the stated operation order.

The definition: a distortion beta on [0, 1], the weight of the levels [0, t], "cvar" min(t / eta, 1) or "wang"
Phi(Phi^-1(t) - eta) (the inverses of IQN's level maps eta tau and Phi(Phi^-1(tau) + eta): eta < 0 is risk-averse).
  quantile rows theta [N]:    Q = sum_j (beta((j+1)/N) - beta(j/N)) theta_j   (index order, levels exact here);
  categorical rows x [Z]:     p = softmax(x), F_k = sum_{k' <= k} p_k', F_{Z-1} = 1, F_{-1} = 0,
                              Q = sum_k (beta(F_k) - beta(F_{k-1})) support_k.
Phi and Phi^-1 are torch.special.ndtr / ndtri in float64 here, checked against the standard library's
statistics.NormalDist (beta_stdlib) by tests/test_risk_host.py.

The error bound of the kernel's fp32 value (absolute, per row), with u = 2^-24 and ulp(x) <= 2u|x|:
  beta at an fp32 input t~ within dt of t:  the input's share is the secant max(beta(t + dt) - beta(t), beta(t) -
      beta(t - dt)) (clamped to [0, 1]; exact for a monotone beta whatever its slope, which for Wang grows without
      bound as t -> 0 at eta < 0 and as t -> 1 at eta > 0); the evaluation's share is u beta for CVaR (one division), and for Wang
      10u beta + phi(z - eta) (10u |z| + u |z - eta|) with z = Phi^-1(t~) -- normcdfinvf and normcdff are each within
      5 ulp (CUDA Math API, single-precision functions), taken at the worst z the input interval allows;
  quantile levels: t = fl32(j / N), dt = u t;  categorical F: e_k = expf(x_k - max x) carries c_k = 4 + |x_k - max x|
      + L_k + max L units of u (expf is within 2 ulp; L the rounding scale of the dueling combination, 0 for plain
      rows), se = sum e and every scan value S_k at most R + 5 roundings (R the atoms per lane), so
      dF_k = u (sum_{k' <= k} p c + F_k (2R + 11 + sum p c)), and 0 at k = Z - 1;
  Q: summation by parts moves an error db_k of beta(F_k) (of beta(t_j)) into Q as db_k |support_{k+1} - support_k|
      (|theta_j-1 - theta_j|); the input rounding of theta adds |w_j| u L_j; the subtraction, product, the lane's R sums
      and the 5 butterfly levels add (R + 7) u sum |w| |support or theta|.
SAFETY doubles the sum; FLOOR keeps a zero bound from demanding bit equality where the arithmetic is not exact."""
import math
from statistics import NormalDist

import torch

import head_ref as R

KINDS = {"cvar": 1, "wang": 2}          # RB_RISK_CVAR, RB_RISK_WANG
U = 2.0 ** -24
ULP_EXP = 2                             # expf
ULP_NORMCDF = 5                         # normcdff
ULP_NORMCDFINV = 5                      # normcdfinvf
SAFETY = 2.0
FLOOR = 2.0 ** -100
BELOW_ONE = 1.0 - 2.0 ** -24            # the largest fp32 below 1
_ND = NormalDist()


def beta_stdlib(t, measure, eta):
    """beta(t) for one float with the standard library's normal distribution."""
    if measure == "cvar":
        return min(t / eta, 1.0)
    if t <= 0.0:
        return 0.0
    if t >= 1.0:
        return 1.0
    return _ND.cdf(_ND.inv_cdf(t) - eta)


def beta(t, measure, eta):
    """beta(t) elementwise in float64."""
    t = t.double()
    if measure == "cvar":
        return (t / eta).clamp(max=1.0)
    return torch.special.ndtr(torch.special.ndtri(t) - eta)


def _phi(y):
    return torch.exp(-0.5 * y * y) / math.sqrt(2.0 * math.pi)


def beta_error(t, dt, measure, eta):
    """Bound of |beta32(t~) - beta(t)| for an fp32 input t~ within dt of t (module docstring)."""
    t, dt = t.double(), dt.double()
    lo, hi = (t - dt).clamp(0.0, 1.0), (t + dt).clamp(0.0, 1.0)
    b = beta(t, measure, eta)
    secant = torch.maximum(beta(hi, measure, eta) - b, b - beta(lo, measure, eta))
    bmax = beta(hi, measure, eta)
    if measure == "cvar":
        return secant + U * bmax
    ev = torch.zeros_like(t)
    for p in (lo, t, hi):
        inner = (p > 0) & (p < 1)
        z = torch.special.ndtri(p.clamp(2.0 ** -149, BELOW_ONE))
        term = _phi(z - eta) * (2 * ULP_NORMCDFINV * U * z.abs() + U * (z - eta).abs())
        ev = torch.maximum(ev, torch.where(inner, term, torch.zeros_like(term)))
    return secant + ev + 2 * ULP_NORMCDF * U * bmax


def _lanes(n):
    return -(-n // 32)


def quantile_values(q, L, measure, eta):
    """Q_beta [..] of quantile rows q [..][N] (float64, known to u L) and its error bound."""
    q, L = q.double(), L.double()
    N = q.shape[-1]
    t = torch.arange(N + 1, dtype=torch.float64, device=q.device) / N
    b = beta(t, measure, eta)
    w = b[1:] - b[:-1]
    Q = (w * q).sum(-1)
    db = beta_error(t, U * t, measure, eta)[1:-1]                    # b_0 = 0 and b_N = 1 are exact
    err = (db * (q[..., :-1] - q[..., 1:]).abs()).sum(-1)
    err = err + (w.abs() * (U * L + (_lanes(N) + 7) * U * q.abs())).sum(-1)
    return Q, SAFETY * err + FLOOR


def categorical_values(x, L, support, measure, eta):
    """Q_beta [..] of logit rows x [..][Z] (float64, known to u L) over a non-decreasing support, and its error bound."""
    x, L = x.double(), L.double()
    s = support.double().to(x.device)
    Z = x.shape[-1]
    Rr = _lanes(Z)
    p = torch.softmax(x, -1)
    F = p.cumsum(-1).clamp(max=1.0)
    F[..., -1] = 1.0
    b = beta(F, measure, eta)
    w = b - torch.nn.functional.pad(b[..., :-1], (1, 0))
    Q = (w * s).sum(-1)
    c = 2 * ULP_EXP + (x - x.max(-1, keepdim=True).values).abs() + L + L.max(-1, keepdim=True).values
    pc = p * c
    dF = U * (pc.cumsum(-1) + F * (2 * Rr + 11 + pc.sum(-1, keepdim=True)))
    dF[..., -1] = 0.0
    db = beta_error(F, dF, measure, eta)[..., :-1]
    err = (db * (s[1:] - s[:-1]).abs()).sum(-1) + (Rr + 7) * U * (w.abs() * s.abs()).sum(-1)
    return Q, SAFETY * err + FLOOR


def values(inp, which, measure, eta):
    """Q_beta [B][A] and bound of the rows c51_ref.logits(inp, which) ("ns": the arg-max's) for inp's entry and kind."""
    import c51_ref as C
    q, L = C.logits(inp, which)
    if "support" in inp:
        return categorical_values(q, L, inp["support"], measure, eta)
    return quantile_values(q, L, measure, eta)


def select_values(z, A, Z, measure, eta, support=None):
    """The select entries' Q_beta [M][A] and bound from head rows z [M][Z + A Z]."""
    q, L = R._dueling(z, A, Z)
    if support is None:
        return quantile_values(q, L, measure, eta)
    return categorical_values(q, L, support, measure, eta)


def astar_ok(Q, err, astar):
    """Rows whose a* is within the bound of the best: Q[a*] >= max Q - (err[a*] + err[argmax])."""
    rows = torch.arange(Q.shape[0], device=Q.device)
    best = Q.argmax(1)
    a = astar.long().to(Q.device)
    return Q[rows, a] >= Q[rows, best] - (err[rows, a] + err[rows, best])


# ---- the stated fp32 order -----------------------------------------------------------------------------------------------
def beta32(t, measure, eta):
    """beta on fp32 tensors, each operation rounded separately (a tensor divisor: torch turns a scalar one into a
    multiplication by its reciprocal)."""
    if measure == "cvar":
        return torch.clamp(t / torch.full_like(t, eta), max=1.0)
    return torch.special.ndtr(torch.special.ndtri(t) - torch.full_like(t, eta))


def _butterfly(s):
    lane = torch.arange(32, device=s.device)
    for o in (16, 8, 4, 2, 1):
        s = s + s[..., lane ^ o]
    return s[..., 0]


def emulate_quantile(x, measure, eta):
    """qr_risk_value of fp32 rows x [..][N] in the kernel's order."""
    N = x.shape[-1]
    Rr = _lanes(N)
    xp = torch.nn.functional.pad(x.float(), (0, 32 * Rr - N))
    j = torch.arange(32 * Rr, device=x.device)
    nn = torch.full((32 * Rr,), float(N), device=x.device)
    lo = beta32(j.float() / nn, measure, eta)
    hi = beta32((j + 1).float() / nn, measure, eta)
    s = torch.zeros(*x.shape[:-1], 32, device=x.device)
    for r in range(Rr):
        sl = slice(32 * r, 32 * (r + 1))
        s = torch.where(j[sl] < N, s + (hi[sl] - lo[sl]) * xp[..., sl], s)
    return _butterfly(s)


def emulate_categorical(x, support, measure, eta):
    """c51_risk_value of fp32 logit rows x [..][Z] over the fp32 support in the kernel's order."""
    Z = x.shape[-1]
    Rr = _lanes(Z)
    dev = x.device
    k = torch.arange(32 * Rr, device=dev)
    xp = torch.nn.functional.pad(x.float(), (0, 32 * Rr - Z), value=-math.inf)
    sp = torch.nn.functional.pad(support.float().to(dev), (0, 32 * Rr - Z))
    mx = xp.max(-1, keepdim=True).values
    e = torch.where(k < Z, torch.exp(xp - mx), torch.zeros_like(xp))
    se = torch.zeros(*x.shape[:-1], 32, device=dev)
    for r in range(Rr):
        se = se + e[..., 32 * r:32 * (r + 1)]
    se = _butterfly(se).unsqueeze(-1)
    lane = torch.arange(32, device=dev)
    carry = torch.zeros(*x.shape[:-1], 1, device=dev)
    b_carry = torch.zeros_like(carry)
    s = torch.zeros(*x.shape[:-1], 32, device=dev)
    for r in range(Rr):
        sl = slice(32 * r, 32 * (r + 1))
        v = e[..., sl]
        for o in (1, 2, 4, 8, 16):
            y = torch.nn.functional.pad(v[..., :-o], (o, 0))
            v = torch.where(lane >= o, v + y, v)
        v = carry + v
        carry = v[..., 31:]
        F = torch.where(k[sl] >= Z - 1, torch.ones_like(v), torch.clamp(v / se.expand_as(v), max=1.0))
        b = beta32(F, measure, eta)
        bp = torch.cat([b_carry, b[..., :-1]], -1)
        b_carry = b[..., 31:]
        s = torch.where(k[sl] < Z, s + (b - bp) * sp[sl], s)
    return _butterfly(s)


def dueling32(z, A, Z):
    """The dueling combination of fp32 head rows z [M][Z + A Z] in the kernels' order: (v + adv) - (sum_a adv) / A."""
    v, adv = z[:, :Z].unsqueeze(1), z[:, Z:].reshape(-1, A, Z)
    acc = torch.zeros_like(v)
    for a in range(A):
        acc = acc + adv[:, a:a + 1]
    return (v + adv) - acc / torch.full_like(acc, float(A))
