"""Float64 reference of value rescaling (Pohlen et al. 2018; DESIGN.md §16) and of the value-rescaled losses behind
rb_c51*_vt_loss_grad, rb_qr*_vt_loss_grad, rb_qr_vt_q_values and rb_learn_stats_batch_qr_vt, built on tests/c51_ref.py
and tests/qr_ref.py (imported, not changed), with a condition scale for every output element.

    h(x)    = sign(x) |x| / (sqrt(|x| + 1) + 1) + eps x
    h^-1(y) = sign(y) d (d + 2),  d = 2|y| / ((1 + 2 eps) + sqrt((1 + 2 eps)^2 + 4 eps |y|))

Both are sums and products of nonnegative terms, so in float64 they are accurate to a few float64 ulp: the reference.

The kernels' fp32 h and h^-1 (u = 2^-24).  h: |x| + 1, sqrt, + 1, the division, eps x and the final sum, six correctly
rounded steps on nonnegative terms; each moves the result by at most 0.5 u relative, sqrt halves its input's, so
|fl(h(x)) - h(x)| <= 4 u |h(x)|.  h^-1: 1 + 2 eps, its square, 4 eps |y|, the sum, sqrt, c + sqrt, the division, d + 2 and
the product: d carries at most 3.5 u, d (d + 2) at most 2 x 3.5 + 1 = 8 u.  The constant c = fl(1 + 2 eps) is itself
rounded once (counted).  So H_U = 8 (in u, relative) bounds either; an input error e moves h by |h'| e (h' = 1 / (2
sqrt(|x| + 1)) + eps <= 1/2 + eps) and h^-1 by |h^-1'| e (h^-1' = 1 / h'(h^-1(y)) <= 2 sqrt(|h^-1(y)| + 1)).  Subnormal
results add at most a few 2^-149 absolute (SUB_FLOOR).

Each stage takes the kernel's result of the stage before (a*, T, m), as c51_ref / qr_ref do, and its scale adds these
terms to the ones those modules derive:
  C51   x_j = r + fl32(s s~_j) (s~ = fl32(h^-1(z_j)) the agent's q_support, an input), Tz_j = h(x_j): b_j carries, in u,
        (h'(x_j) (|r| + 2 |s s~_j|) + H_U |Tz_j| + |Vmin|) / dz in place of (|r| + |s z_j| + |Vmin|) / dz.  The arg-max's
        expected values are c51_ref's with s~ in place of the support.
  QR    x_j = h^-1(q_j) with scale h^-1'(q_j) (L_j + |q_j|) + H_U |x_j| (L the dueling combination's, head_ref._dueling);
        means as qr_ref.means of x; T_j = h(r + s x_j) with scale h'(y_j) (|r| + 2 |s x_j| + |s| scale(x_j)) + H_U |T_j|.
        The loss and gradient are qr_ref.loss_grad's against the kernel's T (in h units, unchanged).
The tolerances stay c51_ref.TAU / qr_ref.TAU (2e-6, 33.5 u) and TAU_EV (1e-6): each added coefficient above is at most
H_U = 8 u per unit of scale, so they keep a margin of 4x.  A slip of the transform (h applied before adding r, eps
dropped, the textbook inverse, the sign lost, h-space arg-max) moves T or a* by a fraction of the value itself."""
import numpy as np
import torch

import c51_ref as C
import head_ref as R
import qr_ref as Q

U = 2.0 ** -24
H_U = 8.0
SUB_FLOOR = 4 * 2.0 ** -149
TAU_H = 2 * H_U * U             # the element-wise h / h^-1 sweeps: 2x the derived bound
EPS_GRID = (0.0, 1e-3, 1e-2)


def h(x, eps):
    ax = x.abs()
    return torch.copysign(ax / ((ax + 1.0).sqrt() + 1.0), x) + eps * x


def hinv(y, eps):
    ay = y.abs()
    c = 1.0 + 2.0 * eps
    d = (2.0 * ay) / (c + (c * c + 4.0 * eps * ay).sqrt())
    return torch.copysign(d * (d + 2.0), y)


def dh(x, eps):
    return 0.5 / (x.abs() + 1.0).sqrt() + eps


def dhinv(y, eps):
    return 1.0 / dh(hinv(y, eps), eps)


def hinv_textbook(y, eps):
    """((sqrt(1 + 4 eps (|y| + 1 + eps)) - 1) / (2 eps))^2 - 1, signed: exact algebra, cancels badly at small |y|."""
    ay = y.abs()
    return torch.copysign((((1.0 + 4.0 * eps * (ay + 1.0 + eps)).sqrt() - 1.0) / (2.0 * eps)) ** 2 - 1.0, y)


def q_support(support, eps):
    """fl32(h^-1(z_j)) from the fp32 support, formed in float64 (as the Agent forms it)."""
    return hinv(support.double(), eps).float()


def h32(x, eps):
    """The kernels' fp32 h (vt_h), step for step in numpy float32 (each operation correctly rounded, as on the device)."""
    x = np.asarray(x, dtype=np.float32)
    ax = np.abs(x)
    r = ax / (np.sqrt(ax + np.float32(1.0)) + np.float32(1.0))
    return np.copysign(r, x) + np.float32(eps) * x


def on_atom_return(support, vmin, dz, k, eps):
    """An fp32 return r of a terminal row whose kernel target lands exactly on atom k, fl32 h(r) == support[k], with
    b = (support[k] - Vmin) / dz an exact integer in fp32, or None: searched over the 32769 fp32 values around
    fl32(h^-1(support[k]))."""
    zk = np.float32(support[k])
    b = (zk - np.float32(vmin)) / np.float32(dz)
    if b != np.floor(b):
        return None
    r0 = np.float32(hinv(torch.tensor(float(zk), dtype=torch.float64), eps))
    bits = np.array(r0, dtype=np.float32).view(np.int32) + np.arange(-16384, 16385, dtype=np.int32)
    cand = bits.view(np.float32)
    hit = np.nonzero(h32(cand, eps) == zk)[0]
    return float(cand[hit[np.argmin(np.abs(hit - 16384))]]) if hit.size else None


# ---- C51 ---------------------------------------------------------------------------------------------------------------
def make_c51_inputs(entry, B, A, Z, eps, seed):
    """c51_ref.make_inputs on the +-10 h-space support, the returns widened to return units: spread rows |r| log-uniform
    in [1e-3, 1e3] with either sign (1 in 8 exactly 0); below / above every target atom at the clamp
    (r beyond h^-1(Vmin / Vmax) by more than s max|s~|); on_atom rows terminal with the kernel's fp32 Tz exactly an atom
    of integer b (on_atom_return; interior atoms where Z > 2), so the fix-ups at an integer b run.  inp["on_atom"] counts
    the on_atom rows that found such a return (the rest keep r = s~_k)."""
    inp = C.make_inputs(entry, B, A, Z, "pm10", seed)
    g = torch.Generator().manual_seed(seed + 1)
    sq = q_support(inp["support"], eps)
    smax = float(sq.abs().max())
    exact = [k for k in range(Z) if (0 < k < Z - 1 or Z == 2)
             and on_atom_return(inp["support"].numpy(), inp["vmin"], inp["dz"], k, eps) is not None]
    hits = 0
    for i in range(B):
        kind = C.RET_KINDS[i % 5]
        u = float(torch.rand(1, generator=g))
        if kind == "spread":
            mag = 10.0 ** (-3.0 + 6.0 * u)
            inp["returns"][i] = 0.0 if i % 8 == 0 else (mag if i % 2 else -mag)
        elif kind == "terminal":
            inp["returns"][i] = (2 * u - 1) * 1e3
        elif kind == "below":
            inp["returns"][i] = float(sq[0]) - C.GAMMA_N * smax - (1.0 + u) * 10.0
        elif kind == "above":
            inp["returns"][i] = float(sq[-1]) + C.GAMMA_N * smax + (1.0 + u) * 10.0
        else:
            inp["returns"][i] = sq[int(u * Z)]
            if exact:
                k = exact[int(u * len(exact))]
                inp["returns"][i] = on_atom_return(inp["support"].numpy(), inp["vmin"], inp["dz"], k, eps)
                hits += 1
    inp.update(eps=eps, support_q=sq, on_atom=hits)
    return inp


def c51_expected_values(inp):
    """ev [B][A] of online(s') over s~ (return units) and its scale."""
    q, L = C.logits(inp, "ns")
    lf = L + (q - q.max(-1, keepdim=True).values).abs()
    return R.expectation(q, lf, inp["support_q"])


def c51_projection(inp, astar):
    """m [B][Z] and its scale for the kernel's a*: c51_ref.projection with Tz_j = h(r + s s~_j) (see the docstring)."""
    Z, eps = inp["Z"], inp["eps"]
    q, L = C.logits(inp, "t")
    pt, _, c, _ = C._softmax_terms(C._row(q, astar), C._row(L, astar))
    sq = C._d(inp["support_q"]).unsqueeze(0)
    r, nt = C._d(inp["returns"]).unsqueeze(1), C._d(inp["nonterminals"]).view(-1, 1)
    vmin, vmax, dz = C.f32(inp["vmin"]), C.f32(inp["vmax"]), C.f32(inp["dz"])
    sc = Q.nonterminal_scale(inp["nonterminals"], inp["gamma_n"]).unsqueeze(1)
    x = r + sc * sq
    tz_raw = h(x, eps)
    tz = tz_raw.clamp(vmin, vmax)
    b = (tz - vmin) / dz
    lo, up = b.floor(), b.ceil()
    lo = torch.where((up > 0) & (lo == up), lo - 1, lo)
    up = torch.where((lo < Z - 1) & (lo == up), up + 1, up)
    m = torch.zeros(b.shape[0], Z + 1, dtype=torch.float64, device=b.device)
    m.scatter_add_(1, lo.long(), pt * (up - b))
    m.scatter_add_(1, up.long(), pt * (b - lo))
    wj = pt * (1 + c + (dh(x, eps) * (r.abs() + 2 * (sc * sq).abs()) + H_U * tz_raw.abs() + abs(vmin)) / dz)
    scale = torch.full((b.shape[0], Z), C.FLOOR, dtype=torch.float64, device=b.device)
    base = b.floor().long()
    for off in range(-2, 3):
        k = base + off
        near = ((k - b).abs() < 1 + C.RHO) & (k >= 0) & (k < Z)
        scale.scatter_add_(1, k.clamp(0, Z - 1), torch.where(near, wj, 0.0))
    return m[:, :Z], scale


# ---- QR ----------------------------------------------------------------------------------------------------------------
QR_CASES = [(32, 6, 51, 1.0), (5, 2, 2, 1.0), (3, 18, 31, 0.25), (33, 6, 32, 10.0), (35, 1, 33, 1.0), (1, 64, 64, 0.25),
            (512, 6, 51, 1.0), (33, 18, 65, 10.0), (5, 6, 128, 1.0), (2048, 6, 51, 0.25), (32, 64, 65, 1.0),
            (512, 18, 128, 1.0)]


def make_qr_inputs(entry, B, A, N, kappa, eps, seed):
    """qr_ref.make_inputs with the spread rows' returns widened to |r| log-uniform in [1e-3, 1e3] (1 in 8 exactly 0)."""
    inp = Q.make_inputs(entry, B, A, N, kappa, seed)
    g = torch.Generator().manual_seed(seed + 1)
    for i in range(0, B, len(Q.ROW_KINDS)):   # the spread rows
        u = float(torch.rand(1, generator=g))
        mag = 10.0 ** (-3.0 + 6.0 * u)
        inp["returns"][i] = 0.0 if i % 8 == 0 else (mag if (i // 6) % 2 else -mag)
    inp["eps"] = eps
    return inp


def hinv_terms(q, L, eps):
    """x = h^-1(q) and its scale (see the docstring)."""
    x = hinv(q, eps)
    return x, dhinv(q, eps) * (L + q.abs()) + H_U * x.abs()


def qr_mean_quantiles(inp):
    """mean_j h^-1(online(s'))_j [B][A] and its scale."""
    q, L = C.logits(inp, "ns")
    x, sx = hinv_terms(q, L, inp["eps"])
    return Q.means(x, sx)


def qr_targets(inp, astar):
    """T = h(r + s h^-1(q_target(s', a*))) [B][N] and its scale, for the kernel's a*."""
    eps = inp["eps"]
    q, L = C.logits(inp, "t")
    x, sx = hinv_terms(C._row(q, astar), C._row(L, astar), eps)
    sc = Q.nonterminal_scale(inp["nonterminals"], inp["gamma_n"]).unsqueeze(1)
    y = C._d(inp["returns"]).unsqueeze(1) + sc * x
    T = h(y, eps)
    r = C._d(inp["returns"]).abs().unsqueeze(1)
    return T, dh(y, eps) * (r + 2 * (sc * x).abs() + sc.abs() * sx) + H_U * T.abs() + Q.FLOOR


def qr_q_values(z, A, N, eps):
    """rb_qr_vt_q_values in float64: mean_j h^-1 of the dueling quantiles [M][A] and its scale."""
    q, L = R._dueling(z, A, N)
    return Q.means(*hinv_terms(q, L, eps))
