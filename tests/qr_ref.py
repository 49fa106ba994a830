"""Float64 reference of the quantile-regression loss (csrc/rb_kernels.cu: k_qr behind rb_qr_loss_grad, k_qr_dueling behind
rb_qr_dueling_loss_grad, k_qr_select behind rb_qr_q_values) with a condition scale for every output element, and the seeded
inputs its tests draw.

The maths (QR-DQN's eq. 10 with IQN's division by kappa): tau_i = (2i + 1) / (2N); theta_i = q_online(s, a)_i;
a* = argmax_a mean_j q_online(s', a)_j; T_j = r + fl32(nt gamma_n) q_target(s', a*)_j; u_ij = T_j - theta_i;
loss = sum_i (1/N) sum_j |tau_i - [u_ij < 0]| H_kappa(u_ij) / kappa; g_i = -(w/B) (1/N) sum_j |tau_i - [u_ij < 0]|
clamp(u_ij, -kappa, kappa) / kappa.  Loss and gradient are continuous in u (at 0 the weight jumps where H and clamp are 0;
at +-kappa H is C1 and clamp continuous), so every bound below is a first-order one; the only discontinuity is a*.

As in tests/c51_ref.py everything is computed from the SAME fp32 tensors the kernel reads, and each stage takes the
kernel's result of the stage before it:
  arg-max   mean_j of every action of online(s'), with scale mean_j (L_j + |q_j|) + |mean| (L the scale of the dueling
            combination, head_ref._dueling; 0 for plain rows): a lane's R <= 4 additions, 5 butterfly levels and the
            division put at most 10 u of it on the kernel's mean.  The kernel's a* is accepted if its mean is within
            TAU_EV (scale[a*] + scale[argmax]) of the best; rows bit-identical across actions must give the first.
  T         from the kernel's a*: |sc q_t| + |T| + |sc| L_t (one product, one sum, the rounding of the dueling
            combination), sc = fl32(nt gamma_n) exactly as the kernel forms it.
  loss, g   from the kernel's T and the float64 theta: u_ij carries at most a few u of D_ij = L_i + |theta_i| + |T_j| + |u_ij|,
            which moves loss by sum tw |clamp(u)| D / (N kappa) and g_i by |w/B| sum_j tw D / (N kappa); the fp32 terms and
            the fixed-order sums (R + 5 levels per row, R + 5 over the rows, two divisions) add at most ~25 u of
            sum tw H / (N kappa) and ~12 u of |w/B| sum tw |clamp| / (N kappa).  So
              loss scale = sum_ij tw (H + |clamp(u)| D) / (N kappa) + FLOOR,
              g scale    = |w/B| (sum_j tw (|clamp(u)| + D) / (N kappa) + FLOOR)   (weight 0: exactly 0),
            and TAU = 2e-6 (33.5 u) covers them.  dz of the dueling entry point: c51_ref.dueling_dz of g.
A slip of the formula (tau_i = i/N, the sign of u, a mean over i, kappa ignored, w/B dropped, the 1/A of dz_a dropped)
moves an element by a fraction of its own size, orders of magnitude above TAU times its scale."""
import numpy as np
import torch

import c51_ref as C
import head_ref as R

TAU_EV = 1e-6
TAU = 2e-6
FLOOR = 2.0 ** -100
GAMMA_N = 0.99 ** 3

# row kinds, cycled over the batch (period 6; weights have period 7, so every combination occurs from B = 42 on)
ROW_KINDS = ("spread", "terminal", "inside", "outside", "const", "ties")
W_PERIOD = 7                              # weight 0 at i % 7 == 3, 1 at i % 7 == 5

# (B, A, N, kappa) of the grid both entry points run (tests/test_gpu_qr_f64.py): N across the R = 2 / R = 4 switch at 64,
# A past the 8 warps, B from 1 to 2048, kappa 0.25, 1 and 10
CASES = [(32, 6, 51, 1.0), (5, 2, 2, 1.0), (3, 18, 31, 0.25), (33, 6, 32, 10.0), (35, 1, 33, 1.0), (1, 64, 64, 0.25),
         (512, 6, 51, 1.0), (33, 18, 65, 10.0), (5, 6, 128, 1.0), (2048, 6, 51, 0.25), (1, 1, 128, 10.0),
         (32, 64, 65, 1.0), (512, 18, 128, 1.0), (42, 2, 2, 0.25), (84, 6, 33, 10.0)]


def _d(t):
    return t.double()


def taus(N, device="cpu"):
    return (2.0 * torch.arange(N, dtype=torch.float64, device=device) + 1.0) / (2.0 * N)


def make_inputs(entry, B, A, N, kappa, seed):
    """Seeded fp32 inputs of one case (CPU tensors), keys as c51_ref.make_inputs (Z = N; no support).  Per row i by
    ROW_KINDS[i % 6]: spread (N(0, 2) rows, r in [-5, 5], nonterminal with probability 0.8); terminal (nt 0); inside
    (rows and r in +-kappa/8: every |u| < kappa); outside (small rows, |r| >= 2 kappa + 7 kappa / 8: every |u| > kappa);
    const (one value per stream row); ties (online(s') rows identical across actions: the first must win).
    Weights U(0.2, 1) with 0 and 1 rows."""
    g = torch.Generator().manual_seed(seed)
    ncol = A * N if entry == "plain" else N + A * N
    kind = torch.arange(B) % len(ROW_KINDS)
    rows = {k: torch.randn(B, ncol, generator=g) * 2.0 for k in ("s", "ns", "t")}
    c = kappa / 8.0
    small = (kind == 2) | (kind == 3)
    for k, t in rows.items():
        t[small] = (torch.rand(int(small.sum()), ncol, generator=g) * 2.0 - 1.0) * c
        blocks = t[kind == 4].view(-1, ncol // N, N)
        t[kind == 4] = blocks[:, :, :1].expand_as(blocks).reshape(-1, ncol)
    ns = rows["ns"][kind == 5]
    first = N if entry == "dueling" else 0
    ns[:, first:] = ns[:, first:first + N].repeat(1, A)
    rows["ns"][kind == 5] = ns
    u = torch.rand(B, generator=g)
    rets = (u * 10.0 - 5.0).float()
    nts = (u < 0.8).float()
    nts[kind == 1] = 0.0
    nts[kind >= 2] = 1.0
    rets[kind == 2] = ((u[kind == 2] * 2.0 - 1.0) * c).float()
    sign = torch.where(torch.arange(B)[kind == 3] % 4 == 3, -1.0, 1.0)
    rets[kind == 3] = (sign * (2.0 * kappa + 7.0 * c + u[kind == 3] * kappa)).float()
    w = torch.rand(B, generator=g) * 0.8 + 0.2
    w[torch.arange(B) % W_PERIOD == 3] = 0.0
    w[torch.arange(B) % W_PERIOD == 5] = 1.0
    acts = torch.randint(0, A, (B,), generator=g)
    inp = dict(entry=entry, B=B, A=A, Z=N, kappa=kappa, gamma_n=GAMMA_N, actions=acts, returns=rets,
               nonterminals=nts.view(B, 1), weights=w)
    if entry == "plain":
        inp.update(q_on_s=rows["s"].view(B, A, N), q_on_ns=rows["ns"].view(B, A, N), q_tg_ns=rows["t"].view(B, A, N))
    else:
        inp.update(z_on=torch.cat([rows["s"], rows["ns"]]), z_tg=rows["t"])
    return inp


def means(q, L):
    """mean_j q [..][A][N] and its scale."""
    ev = q.mean(-1)
    return ev, (L + q.abs()).mean(-1) + ev.abs()


def mean_quantiles(inp):
    """mean [B][A] of online(s') and its scale."""
    return means(*C.logits(inp, "ns"))


def astar_ok(ev, scale, astar):
    best = ev.argmax(1)
    slack = TAU_EV * (C._row(scale, astar) + C._row(scale, best))
    return C._row(ev, astar) >= C._row(ev, best) - slack


def nonterminal_scale(nt, gamma_n):
    """fl32(nt gamma_n), the one place a nonterminal enters (as the kernel forms it), in float64."""
    return _d(nt.view(-1).float() * torch.tensor(np.float32(gamma_n), device=nt.device))


def targets(inp, astar):
    """T [B][N] and its scale, for the kernel's a*."""
    q, L = C.logits(inp, "t")
    qt, lt = C._row(q, astar), C._row(L, astar)
    sc = nonterminal_scale(inp["nonterminals"], inp["gamma_n"]).unsqueeze(1)
    T = _d(inp["returns"]).unsqueeze(1) + sc * qt
    return T, (sc * qt).abs() + T.abs() + sc.abs() * lt + FLOOR


def quantile_terms(theta, T, kappa):
    """(u, tw, H, clamp(u)) [B][N_i][N_j] of online quantiles theta [B][N] against targets T [B][N]."""
    N = theta.shape[1]
    u = T.unsqueeze(1) - theta.unsqueeze(2)
    tau = taus(N, theta.device).view(1, N, 1)
    tw = torch.where(u < 0, 1.0 - tau, tau)
    au = u.abs()
    H = torch.where(au <= kappa, 0.5 * u * u, kappa * (au - 0.5 * kappa))
    return u, tw, H, u.clamp(-kappa, kappa)


def quantile_loss_grad(theta, T, weights, B, kappa):
    """The closed form: (loss [B], g [B][N]) in float64."""
    N = theta.shape[1]
    _, tw, H, cu = quantile_terms(_d(theta), _d(T), kappa)
    loss = (tw * H).sum((1, 2)) / (N * kappa)
    g = -(_d(weights) / B).unsqueeze(1) * (tw * cu).sum(2) / (N * kappa)
    return loss, g


def loss_grad(inp, T):
    """From the kernel's T [B][N]: (loss, scale) [B] and (g, scale) [B][N], the gradient row of the taken action."""
    q, L = C.logits(inp, "s")
    acts, kappa, B = inp["actions"], inp["kappa"], inp["B"]
    theta, lth = C._row(q, acts), C._row(L, acts)
    T = _d(T)
    N = theta.shape[1]
    u, tw, H, cu = quantile_terms(theta, T, kappa)
    D = lth.unsqueeze(2) + theta.abs().unsqueeze(2) + T.abs().unsqueeze(1) + u.abs()
    loss = (tw * H).sum((1, 2)) / (N * kappa)
    loss_scale = (tw * (H + cu.abs() * D)).sum((1, 2)) / (N * kappa) + FLOOR
    wi = (_d(inp["weights"]) / B).unsqueeze(1)
    g = -wi * (tw * cu).sum(2) / (N * kappa)
    g_scale = wi.abs() * ((tw * (cu.abs() + D)).sum(2) / (N * kappa) + FLOOR)
    return (loss, loss_scale), (g, g_scale)


def q_values(z, A, N):
    """rb_qr_q_values in float64: mean quantile [M][A] of z [M][N + A N] and its scale."""
    return means(*R._dueling(z, A, N))
