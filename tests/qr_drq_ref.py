"""Float64 reference of DrQ's K / M averaging under the quantile loss (rb_qr_dueling_avg_loss_grad and its value-rescaled
twin), built stage by stage on tests/qr_ref.py and tests/vt_ref.py, which stay as they are, the way tests/drq_ref.py builds
the categorical one on tests/c51_ref.py.

Target copy k of sample i is the dueling input of qr_ref with online(s') = copy k and target(s') = copy k; a*_k is checked
with qr_ref.astar_ok and T_k (and its scale) taken at the kernel's a*_k, by qr_ref.targets (vt_ref.qr_targets under value
rescaling).  Tbar = mean_k T_k.  From the kernel's Tbar, copy j of s gives loss_j and g_j with qr_ref.loss_grad; loss =
mean_j loss_j, g_j / M, and dz rows through c51_ref.dueling_dz.

Scales.  Each T_k carries its own error within TAU of its scale; the kernel then sums the K rows in k order (K - 1
roundings, each at most u = 2^-24 of a partial sum, so of sum_k |T_k|) and divides by K (one more rounding of |Tbar|):
Tbar is within TAU mean_k scale_k + K u mean_k |T_k|, so its scale is mean_k scale_k + (K u / TAU) mean_k |T_k|.  The loss
likewise: M - 1 roundings of the nonnegative sum and the division add at most M u mean_j loss_j.  The gradient's weight
fl32(w / (M B)) is one rounding, as fl32(w / B) is in the single-copy kernel: no widening.

A slip of the definition (a reversed k sum aside, which only reorders roundings) -- a*_0 for every copy, Tbar without its
1 / K, only copy 0 averaged, the loss not divided by M, w / B in place of w / (M B), the average taken after h^-1 -- moves
some element by a fraction of its own size."""
import torch

import c51_ref as C
import qr_ref as Q
import vt_ref as V

U = 2.0 ** -24


def make_inputs(B, A, N, kappa, seed, M, K, eps=None):
    """qr_ref's dueling inputs (vt_ref's under eps) -- returns, weights, actions and row kinds of copy 0 -- with M online
    copies of s and K copies of s' and of the target rows, each copy drawn from its own seed: z_on [(M + K) B][N + A N],
    z_tg [K B][N + A N]."""
    mk = (lambda s: Q.make_inputs("dueling", B, A, N, kappa, s)) if eps is None else \
        (lambda s: V.make_qr_inputs("dueling", B, A, N, kappa, eps, s))
    src = [mk(seed)] + [mk(seed + 7919 * (c + 1)) for c in range(max(M, K) - 1)]
    inp = dict(src[0])
    inp.update(M=M, K=K, eps=eps, z_on=torch.cat([src[j]["z_on"][:B] for j in range(M)] +
                                                 [src[k]["z_on"][B:] for k in range(K)]),
               z_tg=torch.cat([src[k]["z_tg"] for k in range(K)]))
    return inp


def single(inp, j=0, k=0):
    """qr_ref's dueling input of online copy j and target copy k."""
    B, M = inp["B"], inp["M"]
    d = dict(inp)
    d.update(entry="dueling", z_on=torch.cat([inp["z_on"][j * B:(j + 1) * B], inp["z_on"][(M + k) * B:(M + k + 1) * B]]),
             z_tg=inp["z_tg"][k * B:(k + 1) * B])
    return d


def means(inp):
    """The arg-max's mean quantiles [B][A] of copy 0 and their scale (vt_ref's, of h^-1, under value rescaling)."""
    return Q.mean_quantiles(inp) if inp.get("eps") is None else V.qr_mean_quantiles(inp)


def target(inp, astar):
    """From the kernel's a* [K][B]: (Tbar, scale) [B][N], the per-copy T_k, and whether every a*_k is within the arg-max's
    rounding."""
    K = inp["K"]
    Ts, scales, absT, ok = [], [], [], True
    for k in range(K):
        one = single(inp, 0, k)
        ev, evs = means(one)
        ok = ok and bool(Q.astar_ok(ev, evs, astar[k]).all())
        T, sc = (Q.targets if inp.get("eps") is None else V.qr_targets)(one, astar[k])
        Ts.append(T)
        scales.append(sc)
        absT.append(T.abs())
    widen = (K * U / Q.TAU) * sum(absT) / K
    return sum(Ts) / K, sum(scales) / K + widen, Ts, ok


def loss_dz(inp, Tbar):
    """From the kernel's Tbar [B][N]: (loss, scale) [B], the per-copy losses, and (dz, scale) [M B][N + A N]."""
    M = inp["M"]
    losses, lscales, dzs, dzscales = [], [], [], []
    for j in range(M):
        one = single(inp, j, 0)
        (l, ls), (g, gs) = Q.loss_grad(one, Tbar)
        losses.append(l)
        lscales.append(ls)
        dz, dzs_ = C.dueling_dz(one, g / M, gs / M)
        dzs.append(dz)
        dzscales.append(dzs_)
    loss = sum(losses) / M
    return (loss, sum(lscales) / M + (M * U / Q.TAU) * loss), losses, (torch.cat(dzs), torch.cat(dzscales))


def objective(inp, astar):
    """(loss [B], objective) of the averaged update in float64, differentiable in inp["z_on"]'s rows of s: theta_j of
    online(s_j) at the taken action against Tbar = mean_k T_k (no gradient through the target), loss = mean_j loss_j,
    objective = sum_i w_i loss_i / B.  Written from the definition, not from qr_ref's closed-form gradient."""
    B, A, N, M, K, kappa = inp["B"], inp["A"], inp["Z"], inp["M"], inp["K"], inp["kappa"]
    z = inp["z_on"]
    rows = torch.arange(B, device=z.device)
    with torch.no_grad():
        Tbar = target(inp, astar)[0]
    tau = Q.taus(N, z.device)
    total = 0.0
    for j in range(M):
        zj = z[j * B:(j + 1) * B].double()
        v, a = zj[:, :N].unsqueeze(1), zj[:, N:].view(B, A, N)
        theta = (v + a - a.mean(1, keepdim=True))[rows, inp["actions"].long()]
        u = Tbar.unsqueeze(1) - theta.unsqueeze(2)
        tw = torch.where(u.detach() < 0, 1.0 - tau.view(1, N, 1), tau.view(1, N, 1))
        H = torch.where(u.abs() <= kappa, 0.5 * u * u, kappa * (u.abs() - 0.5 * kappa))
        total = total + (tw * H).sum((1, 2)) / (N * kappa)
    loss = total / M
    return loss, (inp["weights"].double() * loss).sum() / B
