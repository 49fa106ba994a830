"""Float64 reference of Munchausen targets under the quantile loss (rb_qr_dueling_munchausen_loss_grad ->
k_qr_dueling_munchausen, rb_qr_munchausen_loss_grad -> k_qr_munchausen), built on tests/qr_ref.py, which stays as it is.

The definition (DESIGN.md §17): per target row q[A] of mean quantiles, m = max q, S = sum_a exp((q_a - m) / tau),
pi_a = exp((q_a - m) / tau) / S, l_a = (q_a - m) - tau log S; b = alpha max(l_act(s), l0), c_j = sum_a pi_a(s')
(theta_j(s', a) - l_a(s')), T_j = fl32(r + b) + fl32(sc c_j) with sc = fl32(nt gamma_n).  The loss and the gradient are
qr_ref.loss_grad's from the kernel's T.  tau, alpha and l0 enter as the fp32 values the kernel takes.

The error scale of T, derived to first order (u = 2^-24; a basic fp32 operation rounds within u relative; expf is within
2 ulp and logf within 1 ulp (CUDA C Programming Guide, mathematical functions), so within 4u and 2u relative):
  q_a    the kernel's mean quantile, within eq_a = 10 u qs_a (qr_ref.means: the dueling combination, a lane's R additions,
         5 butterfly levels, the division);
  m      within max_a eq_a;   d_a = q_a - m within ed_a = eq_a + e_m + u |d_a|;   x_a = d_a / tau within ed_a / tau + u|x_a|;
  e_a    = exp(x_a) within e_a (ex_a + 4u);   S within sum_a ee_a + (A - 1) u S;   log S within eS / S + 2u |log S|;
  tl     = tau log S within tau elog + u tau log S;   l_a within ed_a + etl + u |l_a|;
  pi_a   within pi_a (ee_a / e_a + eS / S + u);
  b      within alpha el_act + u |b| (clip not binding), u |b| (binding), 2 alpha el_act + u |b| when |l_act - l0| <= el_act:
         there the kernel may take either side of the clip, as astar_ok accepts near-tied arg-maxes;
  c_j    the terms t_a = fl32(pi_a fl32(theta_a - l_a)), theta_a within 3 u Lt_a (the dueling combination's scale), summed in
         action order: within sum_a (epi_a |w_a| + pi_a (3u Lt_a + el_a + u |w_a|) + u |t_a|) + (A - 1) u sum_a |t_a|;
  T_j    within eb + u |r + b| + sc ec_j + u |sc c_j| + u |T_j|.
The dominant term at small tau is pi's sensitivity, epi_a ~ pi_a eq / tau: the scale grows like 1 / tau.  The first-order
bound is doubled for the second-order terms and returned as a scale for qr_ref.TAU, the tolerance every quantile test
uses (scale = 2 bound / TAU).  tests/test_munchausen_host.py checks the bound against an fp32 emulation of the kernel with
expf / logf results moved by up to their documented ulps and the mean quantiles moved by up to their own bound."""
import numpy as np
import torch

import c51_ref as C
import qr_ref as Q

U = 2.0 ** -24
EXP_ULP, LOG_ULP = 2, 1          # CUDA's expf / logf maximum errors in ulp
ALPHA, TEMPERATURE, CLIP = 0.9, 0.03, -1.0
ROW_KINDS = Q.ROW_KINDS + ("wide",)   # qr_ref's, plus target rows whose mean quantiles spread over 3 per action


def _d(t):
    return t.double()


def make_inputs(entry, B, A, N, kappa, seed, alpha=ALPHA, tau=TEMPERATURE, clip=CLIP):
    """qr_ref's inputs for `entry` with the target rows of s added: z_on [B] (s) and z_tg [2B] (s, then s') for "dueling",
    q_on_s, q_tg_s, q_tg_ns [B][A][N] for "plain".  Qr_ref's row kinds for r, nt and w; every seventh row ("wide") has its
    target rows' actions offset by 3 a, so that the clip binds there and pi is nearly one-hot."""
    base = Q.make_inputs(entry, B, A, N, kappa, seed)
    extra = Q.make_inputs(entry, B, A, N, kappa, seed + 7919)
    inp = dict(base, alpha=C.f32(alpha), tau=C.f32(tau), clip=C.f32(clip))
    wide = (torch.arange(B) % len(ROW_KINDS)) == len(ROW_KINDS) - 1
    off = (3.0 * torch.arange(A, dtype=torch.float32)).repeat_interleave(N)
    if entry == "plain":
        t_s, t_ns = extra["q_tg_ns"].clone(), base["q_tg_ns"].clone()
        for t in (t_s, t_ns):
            t.view(B, -1)[wide] += off
        inp.update(q_on_s=base["q_on_s"], q_tg_s=t_s, q_tg_ns=t_ns)
        inp.pop("q_on_ns")
    else:
        t_s, t_ns = extra["z_tg"].clone(), base["z_tg"].clone()
        for t in (t_s, t_ns):
            t[wide, N:] += off
        inp.update(z_on=base["z_on"][:B], z_tg=torch.cat([t_s, t_ns]))
    return inp


def target_logits(inp, which):
    """(q [B][A][N], L) in float64 of the target net on s ("s") or s' ("ns")."""
    B, A, N = inp["B"], inp["A"], inp["Z"]
    if inp["entry"] == "plain":
        q = _d(inp["q_tg_s" if which == "s" else "q_tg_ns"])
        return q, torch.zeros_like(q)
    return C.R._dueling(inp["z_tg"][:B] if which == "s" else inp["z_tg"][B:], A, N)


def online_view(inp):
    """qr_ref's view of the online rows of s (its loss_grad reads "s" only)."""
    if inp["entry"] == "plain":
        return inp
    return dict(inp, z_on=torch.cat([inp["z_on"], inp["z_on"]]))


def policy(q, tau):
    """(pi, l, m, S) of rows q [..][A] in float64: the definition's stable form."""
    m = q.max(-1, keepdim=True).values
    d = q - m
    e = torch.exp(d / tau)
    S = e.sum(-1, keepdim=True)
    return e / S, d - tau * torch.log(S), m, S


def policy_bounds(q, eq, tau):
    """First-order bounds (epi, el) [..][A] on the kernel's pi and l from mean quantiles q within eq (module docstring)."""
    A = q.shape[-1]
    pi, l, m, S = policy(q, tau)
    d = q - m
    em = eq.max(-1, keepdim=True).values
    ed = eq + em + U * d.abs()
    ex = ed / tau + U * (d / tau).abs()
    e = torch.exp(d / tau)
    ee = e * (ex + 2 * EXP_ULP * U)
    eS = ee.sum(-1, keepdim=True) + (A - 1) * U * S
    logS = torch.log(S)
    elog = eS / S + 2 * LOG_ULP * U * logS.abs()
    etl = tau * elog + U * tau * logS.abs()
    el = ed + etl + U * l.abs()
    epi = pi * (ee / e.clamp_min(1e-300) + eS / S + U)
    epi = torch.where(e > 0, epi, ee / S)
    return epi, el


def targets(inp, theta_ns=None):
    """(T [B][N], scale, b [B], b scale, clip_near [B]) in float64 (scale for qr_ref.TAU).  theta_ns [B][A][N] (float64):
    the s' quantiles c_j sums in place of inp's own (pi, l and b still from inp's rows), as the whole-update reference
    takes them."""
    B, A, N = inp["B"], inp["A"], inp["Z"]
    alpha, tau, l0 = inp["alpha"], inp["tau"], inp["clip"]
    qs, Ls = target_logits(inp, "s")
    qn, Ln = target_logits(inp, "ns")
    ev_s, evs_s = Q.means(qs, Ls)
    ev_n, evs_n = Q.means(qn, Ln)
    _, l_s, _, _ = policy(ev_s, tau)
    _, el_s = policy_bounds(ev_s, 10 * U * evs_s, tau)
    pi, l = policy(ev_n, tau)[:2]
    epi, el = policy_bounds(ev_n, 10 * U * evs_n, tau)
    acts = inp["actions"].long()
    la, ela = C._row(l_s, acts), C._row(el_s, acts)
    b = alpha * torch.maximum(la, torch.tensor(l0, dtype=torch.float64))
    near = (la - l0).abs() <= ela
    eb = torch.where(near, 2 * alpha * ela, torch.where(la > l0, alpha * ela, 0.0)) + U * b.abs()
    r = _d(inp["returns"])
    sc = Q.nonterminal_scale(inp["nonterminals"], inp["gamma_n"])
    w = (qn if theta_ns is None else theta_ns) - l.unsqueeze(-1)     # [B][A][N]
    t = pi.unsqueeze(-1) * w
    c = t.sum(1)                                      # [B][N]
    ew = 3 * U * Ln + el.unsqueeze(-1) + U * w.abs()
    et = epi.unsqueeze(-1) * w.abs() + pi.unsqueeze(-1) * ew + U * t.abs()
    ec = et.sum(1) + (A - 1) * U * t.abs().sum(1)
    rb = (r + b).unsqueeze(1)
    T = rb + sc.unsqueeze(1) * c
    err = eb.unsqueeze(1) + U * rb.abs() + sc.unsqueeze(1) * ec + U * (sc.unsqueeze(1) * c).abs() + U * T.abs()
    return T, 2 * err / Q.TAU + Q.FLOOR, b, (2 * eb / Q.TAU + Q.FLOOR), near


def loss_grad(inp, T):
    """From the kernel's T: (loss, scale) [B], (g, scale) [B][N] (qr_ref.loss_grad)."""
    return Q.loss_grad(online_view(inp), T)


def dz(inp, g, gs):
    """dz rows [B][N + A N] and scales of the dueling entry from g."""
    return C.dueling_dz(inp, g, gs)


def grad_rows(inp, g, gs):
    """grad [B][A][N] and scales of the plain entry from g: g at the taken action, exactly 0 elsewhere."""
    B, A, N = inp["B"], inp["A"], inp["Z"]
    full, fs = torch.zeros(B, A, N, dtype=torch.float64), torch.zeros(B, A, N, dtype=torch.float64)
    rows, acts = torch.arange(B), inp["actions"].long().cpu()
    full[rows, acts], fs[rows, acts] = g.cpu(), gs.cpu()
    return full.to(g.device), fs.to(g.device)


def objective(inp):
    """(loss [B], objective) in float64, differentiable in inp["z_on"] (dueling entry): theta of online(s) at the taken
    action against T (no gradient through the target), objective = sum_i w_i loss_i / B.  Written from the definition."""
    B, A, N, kappa = inp["B"], inp["A"], inp["Z"], inp["kappa"]
    with torch.no_grad():
        T = targets(inp)[0]
    z = inp["z_on"].double()
    v, a = z[:, :N].unsqueeze(1), z[:, N:].view(B, A, N)
    theta = (v + a - a.mean(1, keepdim=True))[torch.arange(B), inp["actions"].long()]
    u = T.unsqueeze(1) - theta.unsqueeze(2)
    tau = Q.taus(N, z.device).view(1, N, 1)
    tw = torch.where(u.detach() < 0, 1.0 - tau, tau)
    H = torch.where(u.abs() <= kappa, 0.5 * u * u, kappa * (u.abs() - 0.5 * kappa))
    loss = (tw * H).sum((1, 2)) / (N * kappa)
    return loss, (inp["weights"].double() * loss).sum() / B


# ---- an fp32 emulation of the kernel's scalar stage (numpy), for the bound's host test --------------------------------------
def emulate_fp32(q_s, q_ns, theta_ns, act, r, sc, alpha, tau, l0, rng, wobble=True):
    """One sample's T [N] with the kernel's operation order in numpy fp32, from the mean quantiles q_s, q_ns [A] and the
    s' quantiles theta_ns [A][N] (fp32).  wobble: every expf result moved by a random 0..2 ulp and every logf by 0..1 ulp,
    the documented worst cases."""
    f = np.float32

    def move(x, ulps):
        if not wobble:
            return f(x)
        for _ in range(int(rng.integers(0, ulps + 1))):
            x = np.nextafter(f(x), f(np.inf) if rng.random() < 0.5 else f(-np.inf), dtype=np.float32)
        return f(x)

    def stage(q, act):
        m = q.max()
        S = f(0)
        ds = [f(q[a] - m) for a in range(len(q))]
        es = [move(np.exp(f(d / f(tau)), dtype=np.float32), EXP_ULP) for d in ds]
        for e in es:
            S = f(S + e)
        tl = f(f(tau) * move(np.log(S, dtype=np.float32), LOG_ULP))
        ls = [f(d - tl) for d in ds]
        pis = [f(e / S) for e in es]
        return pis, ls, (ls[act] if act is not None else None)

    _, _, l_act = stage(q_s, act)
    b = f(f(alpha) * max(l_act, f(l0)))
    pis, ls, _ = stage(q_ns, None)
    c = np.zeros(theta_ns.shape[1], np.float32)
    for a in range(len(q_ns)):
        c = (c + (f(pis[a]) * (theta_ns[a] - ls[a]).astype(np.float32)).astype(np.float32)).astype(np.float32)
    return (f(f(r) + b) + (f(sc) * c).astype(np.float32)).astype(np.float32), b
