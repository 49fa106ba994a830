"""Float64 reference of one learner update under Munchausen targets, in tests/update_ref.py's form (its update_ref's
arguments and result), so that tests/test_gpu_update_f64.py's trajectory check runs over it unchanged.

  forward   the online net on the rows of s only (update_ref.net_f64, with the learner's own conv and hidden ReLU sides
            of those rows); the target net's s' quantiles in float64 from its parameters and noise factors;
  target    pi, l and b from the learner's OWN fp32 target rows of [s; s'] (the target head's output the loss kernel
            read), as update_ref takes the learner's own online s' rows for the arg-max: pi's sensitivity to its input
            is 1 / tau, so the float64 forward's difference from the fp32 one would otherwise dominate; the quantiles c_j
            sums stay float64 (munchausen_ref.targets with theta_ns);
  loss      qr_ref.loss_grad against that T, and autograd of sum_i w_i loss_i / B through the float64 online net;
  scale     update_ref's backward of |.| from the loss stage's gradient scale, widened by T's own bound: the kernel forms
            pi, l and T in fp32, within munchausen_ref's derived bound e_T of the float64 T, and g_i moves by at most
            |w / B| sum_j tw_ij e_T,j / (N kappa) with it (the loss by sum_ij tw_ij |clamp(u_ij)| e_T,j / (N kappa)): those
            terms enter the gradient scale over TAU_G and the loss scale over TAU_LOSS."""
import torch

import munchausen_ref as MR
import qr_ref as Q
import update_ref as U


def update_ref(net, P, f_on, x_on, sides, tnet, T, f_tg, x_tg, batch, dist, M=1, K=1, own_ns=None, *, alpha, tau, clip):
    """update_ref.update_ref's contract under Munchausen: x_on's first B rows are s (the online net's only rows), x_tg
    [B] the rows of s', sides the ReLU sides of the online rows of s, own_ns the learner's own fp32 target z rows [2B]
    (s, then s').  No arg-max: ties and alternatives are empty."""
    assert dist == "quantile" and (M, K) == (1, 1)
    B = x_tg.shape[0]
    A, N, kappa = net.action_space, net.atoms, batch["kappa"]
    Pd = {n: t.detach().double().requires_grad_() for n, t in P.items()}
    keep = []
    q_on = U.net_f64(net, Pd, f_on, x_on[:B].double(), sides[0], sides[1], keep=keep)
    with torch.no_grad():
        q_t = U.net_f64(tnet, {n: t.double() for n, t in T.items()}, f_tg, x_tg.double())
    inp = dict(entry="dueling", B=B, A=A, Z=N, z_tg=own_ns, actions=batch["actions"], returns=batch["returns"],
               nonterminals=batch["nonterminals"], weights=batch["weights"], kappa=kappa, gamma_n=batch["gamma_n"],
               alpha=alpha, tau=tau, clip=clip)
    Tq, T_sc, _, _, _ = MR.targets(inp, theta_ns=q_t)
    e_T = T_sc * Q.TAU                        # munchausen_ref's scale is 2 e / TAU: this is twice the derived bound
    plain = dict(inp, entry="plain", q_on_s=q_on.detach())
    (loss, lscale), (g, gs) = Q.loss_grad(plain, Tq)
    rows, acts = torch.arange(B, device=q_on.device), batch["actions"].long()
    theta = q_on.detach()[rows, acts]
    _, tw, _, cu = Q.quantile_terms(theta, Tq, kappa)
    wi = (batch["weights"].double() / B).abs().unsqueeze(1)
    gs = gs + wi * (tw * e_T.unsqueeze(1)).sum(2) / (N * kappa) / U.TAU_G
    lscale = lscale + (tw * cu.abs() * e_T.unsqueeze(1)).sum((1, 2)) / (N * kappa) / U.TAU_LOSS
    g_full, gs_full = torch.zeros_like(q_on), torch.zeros_like(q_on)
    g_full[rows, acts], gs_full[rows, acts] = g, gs
    grads = torch.autograd.grad((q_on * g_full).sum(), list(Pd.values()) + [pre for pre, _ in keep])
    out = dict(loss=loss, lscale=lscale, astar=torch.empty(0, dtype=torch.long), target=(Tq, e_T), ties=[],
               alternatives=[], grads=dict(zip(Pd, grads[:len(Pd)])),
               convs=[(gp, a_in.detach()) for gp, (_, a_in) in zip(grads[len(Pd):], keep)])
    Pa = {n: t.detach().abs().requires_grad_() for n, t in Pd.items()}
    qa = U.net_f64(net, Pa, f_on, x_on[:B].double().abs(), sides[0], sides[1], absolute=True)
    (qa * gs_full).sum().backward()
    out["scales"] = {n: t.grad for n, t in Pa.items()}
    return out
