"""Float64 reference of one learner update (Agent._update_fused / _update_from_batch), built from the stage references:
  forward   conv body + dueling noisy head in float64 from the parameters and noise factors the update used; the conv
            ReLU sides (and, for the whole-update comparison, the hidden ReLU sides) are the learner's own fp32 ones;
  loss      C51's projection (c51_ref) averaged over K target copies and M online copies as drq_ref does, or the quantile
            Huber loss (qr_ref); the double-DQN arg-max is taken on the learner's own fp32 online s' rows, which the loss
            kernel reads, and where the stage tests' astar_ok rule accepts more than one action the update under every
            accepted choice is returned, the learner having to match one of them;
  gradient  float64 autograd of sum_i w_i loss_i / B through the float64 net;
  scale     the same backward with every factor replaced by its absolute value -- |dq| (the loss stage's own gradient
            scale), |W|, |noise factors|, |x|, the learner's masks -- per parameter element: the whole-chain analogue of
            head_ref's and conv_ref's term scales.  |g - g64| <= TAU_G * scale is the bound of the whole update;
  tail      adam_ref.clip_adam / adamw_ref.clip_adamw on the learner's own fp32 flat gradient and state.
TAU_G is derived in tests/test_update_bounds.py and quoted with the H100 observations in DESIGN.md §4."""
import numpy as np
import torch
import torch.nn.functional as F

import adam_ref as AR
import adamw_ref as AWR
import c51_ref as C
import head_ref as R
import qr_ref as Q

TAU_G = 2e-5
TAU_LOSS = 1e-6    # the per-sample loss, of its scale (qr_ref / c51_ref), where it is beyond the north-star 1e-5


def conv_names(net):
    return [(f"convs.{i}.weight", f"convs.{i}.bias") for i, c in enumerate(net.convs) if isinstance(c, torch.nn.Conv2d)]


def net_f64(net, P, f, x, masks=None, hidden_masks=None, absolute=False, keep=None):
    """q [rows][A][Z] of `net` in float64 from parameters P (name -> float64 tensor) and noise factors f (name ->
    (f_in, f_out)).  masks: the conv layers' ReLU sides (else torch.relu); hidden_masks: (fc_h_v's, fc_h_a's) sides.
    absolute: every factor by its absolute value (P and x are passed as such; the noise factors and the dueling
    combination are taken here), for the scale backward.  keep: a list that receives (pre-activation, input) of every
    conv layer."""
    ab = (lambda t: t.abs()) if absolute else (lambda t: t)
    for li, (m, (wn, bn)) in enumerate(zip(net.conv_layers(), conv_names(net))):
        a_in = x
        x = F.conv2d(x, P[wn], P[bn], m.stride, m.padding)
        if keep is not None:
            keep.append((x, a_in))
        x = x * masks[li] if masks is not None else torch.relu(x)
    x = x.reshape(x.shape[0], -1)

    def noisy(name, v):
        fi, fo = (ab(t.double()) for t in f[name])
        w = P[f"{name}.weight_mu"] + P[f"{name}.weight_sigma"] * torch.outer(fo, fi)
        return F.linear(v, w, P[f"{name}.bias_mu"] + P[f"{name}.bias_sigma"] * fo)

    def hidden(name, k):
        h = noisy(name, x)
        return h * hidden_masks[k] if hidden_masks is not None else torch.relu(h)

    A, Z = net.action_space, net.atoms
    v = noisy("fc_z_v", hidden("fc_h_v", 0)).view(-1, 1, Z)
    a = noisy("fc_z_a", hidden("fc_h_a", 1)).view(-1, A, Z)
    if absolute:    # |d q_a / d a_b| = |[a == b] - 1 / A|
        return v + a * (1.0 - 2.0 / A) + a.sum(1, keepdim=True) / A
    return v + a - a.mean(1, keepdim=True)


def f64_forward(net, P, f, x):
    """q [rows][A][Z] of `net` in float64 from parameters P (name -> float64 tensor) and its noise factors f."""
    return net_f64(net, P, f, x)


def f64_forward_masked(net, P, f, x, masks):
    """f64_forward with each conv ReLU replaced by the fp32 forward's side: a pre-activation within rounding of zero can
    land on the other side in float64, and that one activation's gradient then shows in the conv gradients (DESIGN.md
    §4); taking the learner's sides leaves only the arithmetic to compare."""
    return net_f64(net, P, f, x, masks)


def f64_projection(ag, q_t, r, nt, gamma_n=None):
    """m [B][Z] of softmax(q_t) with agent.py:79-92's arithmetic in float64 (fp32 arguments as the kernel gets them);
    gamma_n None: the agent's fixed discount ** n."""
    Z = ag.atoms
    s = ag.support.double().unsqueeze(0)
    gn = ag.discount ** ag.n if gamma_n is None else gamma_n
    vmin, vmax, dz, gn = (C.f32(v) for v in (ag.Vmin, ag.Vmax, ag.delta_z, gn))
    pt = torch.softmax(q_t, 1)
    b = ((r.unsqueeze(1) + nt.view(-1, 1) * gn * s).clamp(vmin, vmax) - vmin) / dz
    lo, up = b.floor(), b.ceil()
    lo = torch.where((up > 0) & (lo == up), lo - 1, lo)
    up = torch.where((lo < Z - 1) & (lo == up), up + 1, up)
    m = torch.zeros(b.shape[0], Z + 1, dtype=torch.float64, device=b.device)
    m.scatter_add_(1, lo.long(), pt * (up - b))
    m.scatter_add_(1, up.long(), pt * (b - lo))
    return m[:, :Z]


def qr_objective(q_s, q_ns, q_t, actions, returns, nonterminals, weights, gamma_n, kappa):
    """(per-sample loss, objective) of the quantile loss in float64 (differentiable in q_s); nonterminals enter only as
    fl32(nt gamma_n), as in the kernels."""
    B, _, N = q_s.shape
    rows = torch.arange(B, device=q_s.device)
    theta = q_s[rows, actions]
    with torch.no_grad():
        best = q_ns.mean(2).argmax(1)
        sc = (nonterminals.view(-1).float() * torch.tensor(np.float32(gamma_n), device=q_s.device)).double()
        T = returns.double().unsqueeze(1) + sc.unsqueeze(1) * q_t[rows, best]
    u = T.unsqueeze(1) - theta.unsqueeze(2)
    tau = (2.0 * torch.arange(N, dtype=torch.float64, device=q_s.device) + 1.0) / (2.0 * N)
    tw = torch.where(u.detach() < 0, 1.0 - tau.view(1, N, 1), tau.view(1, N, 1))
    au = u.abs()
    H = torch.where(au <= kappa, 0.5 * u * u, kappa * (au - 0.5 * kappa))
    loss = (tw * H).sum((1, 2)) / (N * kappa)
    return loss, (weights.double() * loss).sum() / B


# ---- the whole update ----------------------------------------------------------------------------------------------------
MAX_TIE_CHOICES = 16


def own_ns_logits(z, A, Z):
    """(q, L) [rows][A][Z] of the learner's own fp32 head output rows z [rows][Z(1 + A)]: the dueling combination in
    float64 and its rounding scale, as c51_ref / qr_ref take the kernel's inputs."""
    return R._dueling(z, A, Z)


def argmax_choices(q, L, dist, support=None):
    """The double-DQN arg-max over the learner's own online s' logits q [B][A][Z] (known to L): (arg-max [B], ties), ties
    = [(row, [actions astar_ok accepts])] for the rows where the stage tests' rule accepts more than one action."""
    if dist == "quantile":
        ev, evs = Q.means(q, L)
        ok_rule = Q.astar_ok
    else:
        ev, evs = R.expectation(q, L + (q - q.max(-1, keepdim=True).values).abs(), support)
        ok_rule = C.astar_ok
    B, A = ev.shape
    best = ev.argmax(1)
    ok = torch.stack([ok_rule(ev, evs, torch.full((B,), a, dtype=torch.long, device=ev.device)) for a in range(A)], 1)
    ties = [(i, torch.nonzero(ok[i]).view(-1).tolist()) for i in torch.nonzero(ok.sum(1) > 1).view(-1).tolist()]
    return best, ties


def loss_stage(q_on, q_t, batch, dist, M, K, astars):
    """The loss of the update from float64 online rows q_on [(M + K) B][A][Z] (M copies of s, then K of s', copy-major),
    target rows q_t [K B][A][Z] and the arg-max of every target copy, astars [K][B].  batch: dict(actions, returns,
    nonterminals, weights, gamma_n, and support, vmin, vmax, dz for "categorical" or kappa for "quantile").  Returns
    dict(loss [B], lscale [B], g [M B][A][Z] = d objective / d q of the s rows, gs = its scale, astar, target (m or T and
    its scale))."""
    q_on, q_t = q_on.detach(), q_t.detach()
    B, A, Z = q_t.shape[0] // K, q_t.shape[1], q_t.shape[2]
    rows = torch.arange(B, device=q_on.device)
    base = dict(batch, B=B, A=A, Z=Z, entry="plain")
    tg = []
    for k in range(K):
        inp = dict(base, q_on_ns=q_on[(M + k) * B:(M + k + 1) * B], q_tg_ns=q_t[k * B:(k + 1) * B])
        tg.append(Q.targets(inp, astars[k]) if dist == "quantile" else C.projection(inp, astars[k]))
    t, ts = sum(x[0] for x in tg) / K, sum(x[1] for x in tg) / K
    out = dict(loss=0.0, lscale=0.0, g=[], gs=[], astar=torch.stack(list(astars)), target=(t, ts))
    for j in range(M):
        inp = dict(base, q_on_s=q_on[j * B:(j + 1) * B])
        (l, ls), (g, gs) = (Q.loss_grad if dist == "quantile" else C.loss_grad)(inp, t)
        full, fs = torch.zeros_like(q_on[:B]), torch.zeros_like(q_on[:B])
        full[rows, batch["actions"]], fs[rows, batch["actions"]] = g / M, gs / M
        out["loss"], out["lscale"] = out["loss"] + l / M, out["lscale"] + ls / M
        out["g"].append(full)
        out["gs"].append(fs)
    out["g"], out["gs"] = torch.cat(out["g"]), torch.cat(out["gs"])
    return out


def update_ref(net, P, f_on, x_on, sides, tnet, T, f_tg, x_tg, batch, dist, M=1, K=1, own_ns=None):
    """One update in float64.  P / T: online / target parameters (name -> tensor of any float type), f_on / f_tg their
    noise factors, x_on [(M + K) B] online rows, x_tg [K B] target rows, sides = (conv masks, hidden masks) of the online
    rows (the learner's own).  own_ns: (q, L) [K B][A][Z] of the learner's own online s' logits, which the loss kernel's
    arg-max reads (None: the float64 rows).  Returns dict(loss, lscale, astar, target, grads {name: float64}, scales
    {name: float64}, convs [(d objective / d pre-activation, input activation)] per conv layer (for
    conv_ref.wgrad_normwise), ties [(copy, row, accepted actions)], alternatives [dict(loss, lscale, astar, grads)]: the
    update under every other choice of the tied rows' actions)."""
    B = x_tg.shape[0] // K
    Pd = {n: t.detach().double().requires_grad_() for n, t in P.items()}
    keep = []
    q_on = net_f64(net, Pd, f_on, x_on.double(), sides[0], sides[1], keep=keep)
    with torch.no_grad():
        q_t = net_f64(tnet, {n: t.double() for n, t in T.items()}, f_tg, x_tg.double())
    if own_ns is None:
        own_ns = (q_on[M * B:].detach(), torch.zeros_like(q_on[M * B:]))
    best, ties = [], []
    for k in range(K):
        bk, tk = argmax_choices(own_ns[0][k * B:(k + 1) * B], own_ns[1][k * B:(k + 1) * B], dist, batch.get("support"))
        best.append(bk)
        ties += [(k, i, acts) for i, acts in tk]
    choices = [dict()]
    for k, i, acts in ties:
        choices = [dict(c, **{f"{k},{i}": a}) for c in choices for a in acts]
    if len(choices) > MAX_TIE_CHOICES:
        raise AssertionError(f"{len(ties)} near-tied arg-max rows: more choices than the reference enumerates")
    outs = []
    for c in choices:
        astars = [b.clone() for b in best]
        for key, a in c.items():
            k, i = map(int, key.split(","))
            astars[k][i] = a
        o = loss_stage(q_on, q_t, batch, dist, M, K, astars)
        grads = torch.autograd.grad((q_on[:M * B] * o["g"]).sum(), list(Pd.values()) + [pre for pre, _ in keep],
                                    retain_graph=True)
        o["grads"] = dict(zip(Pd, grads[:len(Pd)]))
        o["convs"] = [(g[:M * B], a_in[:M * B].detach()) for g, (_, a_in) in zip(grads[len(Pd):], keep)]
        outs.append(o)
    out = next(o for o, c in zip(outs, choices) if all(c[key] == int(best[int(key.split(",")[0])][int(key.split(",")[1])])
                                                       for key in c))
    out["ties"] = ties
    out["alternatives"] = [o for o in outs if o is not out]
    # the scale: the same backward on |P|, |f|, |x| with the same sides, started from the loss stage's gradient scale
    # (the tied choices change g, not its scale's terms beyond the rounding the stage rule allows)
    Pa = {n: t.detach().abs().requires_grad_() for n, t in Pd.items()}
    s_masks = [m[:M * B] for m in sides[0]]
    s_hidden = [m[:M * B] for m in sides[1]]
    qa = net_f64(net, Pa, f_on, x_on[:M * B].double().abs(), s_masks, s_hidden, absolute=True)
    (qa * out["gs"]).sum().backward()
    out["scales"] = {n: t.grad for n, t in Pa.items()}
    return out


def flat(named, net, offsets, numel, device):
    """{name: tensor} laid out as the optimiser's flat buffer (float64, padding 0)."""
    g = torch.zeros(numel, dtype=torch.float64, device=device)
    for (n, _), off in zip(net.named_parameters(), offsets):
        g[off:off + named[n].numel()] = named[n].reshape(-1).double()
    return g


def optimiser_ref(opt, before, flat_grad):
    """The optimiser step the learner took, in float64, from its own state before the step and its own fp32 flat
    gradient: adam_ref.clip_adam, or adamw_ref.clip_adamw under the group optimiser.  before: dict(flat_param, exp_avg,
    exp_avg_sq, step_count, group_steps [ENCODER, HEAD])."""
    if opt.grouped:
        groups = [(b, e, opt.weight_decay) for b, e in opt.groups]
        return AWR.clip_adamw(before["flat_param"], flat_grad, before["exp_avg"], before["exp_avg_sq"], groups,
                              before["group_steps"], 1.0, opt.max_norm, opt.lr, opt.betas[0], opt.betas[1], opt.eps)
    return AR.clip_adam(before["flat_param"], flat_grad, before["exp_avg"], before["exp_avg_sq"], before["step_count"], 1.0,
                        opt.max_norm, opt.lr, opt.betas[0], opt.betas[1], opt.eps)


def ratio(got, ref, scale):
    """Largest |got - ref| / scale over a tensor (an element of scale 0 must be exact)."""
    err = (got.double() - ref).abs()
    r = torch.where(scale > 0, err / scale.clamp_min(1e-300), torch.where(err > 0, float("inf"), 0.0))
    return float(r.max()) if r.numel() else 0.0
