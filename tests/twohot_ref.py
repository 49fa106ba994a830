"""Float64 reference of two-hot targets for the categorical loss (rb_c51_twohot_loss_grad -> k_c51_twohot,
rb_c51_dueling_twohot_loss_grad -> k_c51_dueling_twohot and their _vt twins), built on tests/c51_ref.py, tests/vt_ref.py
and tests/hlg_ref.py, which stay as they are.

The definition (DESIGN.md §21): a* is the double-DQN arg-max (c51_ref.expected_values, or vt_ref.c51_expected_values over
s~ = support_q under value rescaling, accepted by c51_ref.astar_ok); ybar the expected value of target(s') at a* over the
same support; x = r + sc ybar with sc = fl32(nt gamma_n); y = clamp(x, Vmin, Vmax), or clamp(h(x), Vmin, Vmax) under the
transform; b = (y - Vmin) / dz with the kernel's fp32 Vmin and dz; l = floor(b), u = ceil(b) with C51's two fix-ups;
m_l = u - b, m_u = b - l, every other m_k = 0, and an index u = Z (rounding puts b past Z - 1) dropped as c51_ref drops it.
So m_k = max(0, 1 - |k - b|): continuous and piecewise linear in y, |dm_k/dy| <= 1 / dz.  The loss and the gradient are
c51_ref.loss_grad's against m (hlg_ref.loss_grad folds m's bound in).

First-order error bound of the kernel's y and m against this reference (u = 2^-24, a basic fp32 operation rounds within
u relative):
  ybar   within c51_ref.TAU_EV times head_ref.expectation's scale of the target row at a* (hlg_ref.ybar's bound);
  x      fl32(r + fl32(sc ybar)): within ex = sc e_ybar + u |sc ybar| + u |x|;
  y      off: ey = ex (the clamp does not add to it); under the transform ey = h'(x) ex + H_U u |h(x)| (vt_ref's bound of
         the fp32 h);
  b      fl32(fl32(y - Vmin) / dz): the two roundings, eb = u (|y - Vmin| / dz + |b|);
  m_k    fl32(u - b) or fl32(b - l): em_k = eb + u m_k + ey / dz on the atoms within 1 + RHO of b (every other atom is
         exactly 0 in both), the last term |dm/dy| ey;
  loss, grad  from m: hlg_ref.loss_grad, c51_ref's loss-row tolerance plus what em moves.
Each first-order bound is doubled for the second-order terms, and every bound carries c51_ref.FLOOR.
tests/test_two_hot_host.py checks the bounds against an fp32 emulation of the stated operation order with ybar moved by up
to its own bound."""
import numpy as np
import torch

import c51_ref as C
import head_ref as R
import hlg_ref as H
import vt_ref as V

U = 2.0 ** -24
EPS_GRID = (1e-3, 0.0)          # the transform's eps on the kernel grid


def make_inputs(entry, B, A, Z, sup_kind, seed, eps=None):
    """c51_ref's inputs (eps given: value rescaling, with support_q = fl32(h^-1(support)) and eps), with rows moved:
    i % 11 == 6 terminal with y exactly on an atom (r = z_k; under the transform a return whose fp32 h is z_k, where one
    exists), i % 11 == 9 terminal far below Vmin and i % 11 == 10 terminal far above Vmax (clamped to them)."""
    inp = C.make_inputs(entry, B, A, Z, sup_kind, seed)
    sup = inp["support"]
    if eps is not None:
        inp.update(eps=eps, support_q=V.q_support(sup, eps))
    far = 1e6 if eps is None else 1e12
    g = torch.Generator().manual_seed(seed + 23)
    for i in range(B):
        if i % 11 == 6:
            k = int(torch.randint(0, Z, (1,), generator=g))
            r = float(sup[k])
            if eps is not None:
                r = V.on_atom_return(sup.numpy(), inp["vmin"], inp["dz"], k, eps)
                r = float(inp["support_q"][k]) if r is None else r
            inp["returns"][i], inp["nonterminals"][i] = r, 0.0
        elif i % 11 in (9, 10):
            inp["returns"][i], inp["nonterminals"][i] = (-far if i % 11 == 9 else far), 0.0
    return inp


def support_ev(inp):
    """The support the expected values take: s~ under the transform, else the support."""
    return inp["support_q"] if "eps" in inp else inp["support"]


def expected_values(inp):
    """ev [B][A] of online(s') over support_ev and its scale."""
    return V.c51_expected_values(inp) if "eps" in inp else C.expected_values(inp)


def ybar(inp, astar):
    """(ybar, bound) [B]: the expected value of target(s') at a* over support_ev, and the kernel's error bound on it."""
    q, L = C.logits(inp, "t")
    q, L = C._row(q, astar.cpu()), C._row(L, astar.cpu())
    lf = L + (q - q.max(-1, keepdim=True).values).abs()
    ev, scale = R.expectation(q.unsqueeze(1), lf.unsqueeze(1), support_ev(inp).cpu())
    return ev[:, 0], C.TAU_EV * scale[:, 0]


def split(y, vmin, dz, Z):
    """(m [B][Z], b [B]) of y [B] (float64) by the stated rule: b = (y - vmin) / dz, floor / ceil, the fix-ups, m_l = u - b
    and m_u = b - l, an index u = Z dropped."""
    b = (y - vmin) / dz
    lo, up = b.floor(), b.ceil()
    lo = torch.where((up > 0) & (lo == up), lo - 1, lo)
    up = torch.where((lo < Z - 1) & (lo == up), up + 1, up)
    m = torch.zeros(b.shape[0], Z + 1, dtype=torch.float64)      # column Z: the dropped part
    m.scatter_add_(1, lo.long().unsqueeze(1), (up - b).unsqueeze(1))
    m.scatter_add_(1, up.long().unsqueeze(1), (b - lo).unsqueeze(1))
    return m[:, :Z], b


def target(inp, astar, y=None):
    """(y, ey) [B] and (m, em) [B][Z] for the kernel's a*.  y given (the kernel's): m is formed from it, and em leaves out
    the y term (the caller checks y on its own)."""
    Z = inp["Z"]
    r = C._d(inp["returns"].reshape(-1).cpu())
    sc = H.sc_of(inp)
    yb, eyb = ybar(inp, astar)
    x = r + sc * yb
    ex = sc * eyb + U * (sc * yb).abs() + U * x.abs()
    vmin, vmax, dz = C.f32(inp["vmin"]), C.f32(inp["vmax"]), C.f32(inp["dz"])
    if "eps" in inp:
        hx = V.h(x, inp["eps"])
        ey1 = V.dh(x, inp["eps"]) * ex + V.H_U * U * hx.abs()
    else:
        hx, ey1 = x, ex
    # a target clamped by more than its error is Vmin / Vmax exactly
    ey1 = torch.where((hx - 2 * ey1 > vmax) | (hx + 2 * ey1 < vmin), 0.0, ey1)
    y64 = hx.clamp(vmin, vmax)
    ey = 2 * ey1 + C.FLOOR
    if y is not None:
        y64 = C._d(y.reshape(-1).cpu())
    m, b = split(y64, vmin, dz, Z)
    eb = U * ((y64 - vmin).abs() / dz + b.abs())
    em = eb.unsqueeze(1) + U * m
    width = torch.full_like(b, 1 + C.RHO)
    if y is None:
        em = em + (ey1 / dz).unsqueeze(1)
        width = width + 2 * ey1 / dz
    k = torch.arange(Z, dtype=torch.float64).unsqueeze(0)
    near = (k - b.unsqueeze(1)).abs() < width.unsqueeze(1)
    return (y64, ey), (m, torch.where(near, 2 * em, 0.0) + C.FLOOR)


loss_grad = H.loss_grad
