"""Float64 reference of HL-Gauss targets for the categorical loss (rb_c51_dueling_hlg_loss_grad -> k_c51_dueling_hlg,
rb_c51_hlg_loss_grad -> k_c51_hlg), built on tests/c51_ref.py, which stays as it is.

The definition (DESIGN.md §20): a* is the double-DQN arg-max (c51_ref.expected_values, accepted by c51_ref.astar_ok);
ybar the expected value of target(s') at a*; y = clamp(r + sc ybar, Vmin, Vmax) with sc = fl32(nt gamma_n); bin k is
[e_k, e_{k+1}], e_k = fl32(z_k - h) for k < Z and e_Z = fl32(z_{Z-1} + h), h = fl32(dz / 2); t_k = (e_k - y) c with the
kernel's c = fl32(1 / fl32(fl32(sqrt 2) sigma)); u_k = the mass of the unit-variance erf between t_k and t_{k+1},
m_k = u_k / sum_j u_j.  The loss and the gradient are c51_ref.loss_grad's against m.

First-order error bound of the kernel's y and m against this reference (u = 2^-24, a basic fp32 operation rounds within
u relative; erff is within 2 ulp, erfcf within 4, expf within 2 and logf within 1 (CUDA Math API, single-precision
functions), and an ulp of v is at most 2u |v|):
  ybar   within c51_ref.TAU_EV times head_ref.expectation's scale of the target row at a*;
  y      fl32(r + fl32(sc ybar)): within ey = sc e_ybar + u |sc ybar| + u |r + sc ybar| (the clamp does not add to it);
  t_k    fl32(fl32(e_k - y) c): et_k = 2u |t_k| from the roundings (y's error is carried by the sensitivity below);
  u_k    1/2 (f(a) - f(b)) with f = erfc or erf: eu_k = 1/2 (E(a) + E(b)) + u u_k + (1/sqrt(pi)) sum_{t in t_k, t_{k+1}}
         exp(-t^2) et, with E = 2u ulps |f| (erfcf's 4 ulp on the tails, erff's 2 ulp in the bin holding y);
  U      positive terms, each lane over at most 4 atoms, then 5 butterfly levels: eU = sum eu_j + 9u U;
  m_k    fl32(u_k / U): em_k = (eu_k + m_k eU) / U + u m_k + |dm_k/dy| ey, the sensitivity bounded by
         |dm_k/dy| <= (g_k + m_k sum_j g_j) / U, g_k = (c / sqrt(pi)) (exp(-t_k^2) + exp(-t_{k+1}^2)) -- with
         t = (e - y) / (sqrt(2) sigma) that is (phi(t'_k) + phi(t'_{k+1})) / (sqrt(2) sigma U) and more, phi the standard
         normal density at t' = sqrt(2) t, up to the factor sqrt(2) of the two conventions.
  loss, grad  from m: the kernel's m is within em, so the loss moves by sum |log p| em and g by (w/B)(p sum em + em); the
         loss row's own arithmetic is c51_ref's (TAU times its scale).
Each first-order bound is doubled for the second-order terms, and every bound carries c51_ref.FLOOR.
tests/test_hl_gauss_host.py checks the bounds against an fp32 emulation of the stated operation order with every
erff / erfcf result moved by up to its documented ulps and ybar moved by up to its own bound."""
import math

import numpy as np
import torch

import c51_ref as C
import head_ref as R

U = 2.0 ** -24
ERF_ULP, ERFC_ULP = 2, 4          # CUDA's erff / erfcf maximum errors in ulp
RATIOS = (0.1, 0.75, 4.0)        # sigma / dz of the kernel grid
SQRT2_F32 = float(np.float32(math.sqrt(2.0)))


def _d(t):
    return t.double()


def sigma_of(ratio, dz):
    """The sigma the agent passes the kernels: fl32(ratio dz)."""
    return C.f32(ratio * dz)


def c_of(sigma):
    """c = fl32(1 / fl32(fl32(sqrt 2) sigma)), the fp32 the kernel forms."""
    s = np.float32(SQRT2_F32) * np.float32(sigma)
    return float(np.float32(1.0) / np.float32(s))


def edges(support, dz):
    """e [Z + 1] in float64 holding the kernel's fp32 edges: fl32(z_k - h), k < Z, and fl32(z_{Z-1} + h)."""
    s = support.cpu().numpy().astype(np.float32)
    h = np.float32(dz) * np.float32(0.5)
    e = np.concatenate([s - h, s[-1:] + h]).astype(np.float32)
    return torch.from_numpy(e.astype(np.float64))


def make_inputs(entry, B, A, Z, sup_kind, seed, ratio):
    """c51_ref's inputs plus sigma, with rows i % 11 == 6 moved onto a bin edge (nt 0, r = e_k exactly) and rows
    i % 11 == 9 onto an atom (nt 0, r = z_k)."""
    inp = C.make_inputs(entry, B, A, Z, sup_kind, seed)
    e = edges(inp["support"], inp["dz"])
    g = torch.Generator().manual_seed(seed + 17)
    for i in range(B):
        if i % 11 in (6, 9):
            k = int(torch.randint(0, Z + 1 if i % 11 == 6 else Z, (1,), generator=g))
            inp["returns"][i] = float(e[k]) if i % 11 == 6 else float(inp["support"][k])
            inp["nonterminals"][i] = 0.0
    inp["sigma"] = sigma_of(ratio, inp["dz"])
    return inp


def sc_of(inp):
    """sc = fl32(nt gamma_n) [B] in float64."""
    nt = inp["nonterminals"].reshape(-1).cpu().numpy().astype(np.float32)
    return torch.from_numpy((nt * np.float32(inp["gamma_n"])).astype(np.float64))


def ybar(inp, astar):
    """(ybar, bound) [B]: the expected value of target(s') at a* and the kernel's error bound on it."""
    q, L = C.logits(inp, "t")
    q, L = C._row(q, astar.cpu()), C._row(L, astar.cpu())
    lf = L + (q - q.max(-1, keepdim=True).values).abs()
    ev, scale = R.expectation(q.unsqueeze(1), lf.unsqueeze(1), inp["support"].cpu())
    return ev[:, 0], C.TAU_EV * scale[:, 0]


def _erf_terms(t):
    """(u, the erff / erfcf error term E(a) + E(b)) per bin from the edge values t [B][Z + 1], by the kernel's cases."""
    t0, t1 = t[:, :-1], t[:, 1:]
    above, below = t0 >= 0, t1 <= 0
    erfc = torch.special.erfc
    u_above = 0.5 * (erfc(t0) - erfc(t1))
    u_below = 0.5 * (erfc(-t1) - erfc(-t0))
    u_mid = 0.5 * (torch.erf(t1) - torch.erf(t0))
    u = torch.where(above, u_above, torch.where(below, u_below, u_mid))
    ea = 2 * U * ERFC_ULP * (erfc(t0) + erfc(t1))
    eb = 2 * U * ERFC_ULP * (erfc(-t1) + erfc(-t0))
    em = 2 * U * ERF_ULP * (torch.erf(t1).abs() + torch.erf(t0).abs())
    return u, torch.where(above, ea, torch.where(below, eb, em))


def target(inp, astar, y=None):
    """(y, ey) [B] and (m, em) [B][Z] for the kernel's a*.  y given (the kernel's): m is formed from it, and em leaves out
    the y term (the caller checks y on its own)."""
    r = _d(inp["returns"].reshape(-1).cpu())
    sc = sc_of(inp)
    yb, eyb = ybar(inp, astar)
    raw = r + sc * yb
    y64 = raw.clamp(C.f32(inp["vmin"]), C.f32(inp["vmax"]))
    ey = 2 * (sc * eyb + U * (sc * yb).abs() + U * raw.abs()) + C.FLOOR
    if y is not None:
        y64 = _d(y.reshape(-1).cpu())
    c = c_of(inp["sigma"])
    e = edges(inp["support"], inp["dz"]).unsqueeze(0)
    t = (e - y64.unsqueeze(1)) * c
    u, e_erf = _erf_terms(t)
    et = 2 * U * t.abs()
    dens = torch.exp(-t * t)
    eu = 0.5 * e_erf + U * u + (dens[:, :-1] * et[:, :-1] + dens[:, 1:] * et[:, 1:]) / math.sqrt(math.pi)
    Us = u.sum(1, keepdim=True)
    m = u / Us
    eU = eu.sum(1, keepdim=True) + 9 * U * Us
    g = c / math.sqrt(math.pi) * (dens[:, :-1] + dens[:, 1:])
    dmdy = (g + m * g.sum(1, keepdim=True)) / Us
    em = (eu + m * eU) / Us + U * m
    if y is None:
        em = em + dmdy * ey.unsqueeze(1)
    return (y64, ey), (m, 2 * em + C.FLOOR)


def masses_ndtr(y, sigma, e):
    """m [B][Z] by an independent float64 formula: differences of the normal CDF (scipy.special.ndtr) over the edges,
    each bin taken on the side of y where the CDF's tail keeps its accuracy, normalised by the mass in [e_0, e_Z]."""
    from scipy.special import ndtr
    y, e = np.asarray(y, np.float64)[:, None], np.asarray(e, np.float64)[None, :]
    a, b = (e[:, :-1] - y) / sigma, (e[:, 1:] - y) / sigma
    mass = np.where(a >= 0, ndtr(-a) - ndtr(-b), ndtr(b) - ndtr(a))
    return mass / mass.sum(1, keepdims=True)


def loss_grad(inp, m, em):
    """(loss, bound) [B] and (g, bound) [B][Z] of the reference m with em folded in: c51_ref.loss_grad against m, the
    bound C.TAU times its scale plus what em moves."""
    (loss, ls), (g, gs) = C.loss_grad(inp, m)
    q, L = C.logits(inp, "s")
    acts = inp["actions"].cpu()
    p, logp, _, _ = C._softmax_terms(C._row(q, acts), C._row(L, acts))
    wi = (_d(inp["weights"].cpu()) / inp["B"]).unsqueeze(1)
    el = (logp.abs() * em).sum(1)
    eg = wi.abs() * (p * em.sum(1, keepdim=True) + em)
    return (loss, C.TAU * ls + 2 * el), (g, C.TAU * gs + 2 * eg)
