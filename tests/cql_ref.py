"""Float64 reference of CQL(H)'s regulariser (DESIGN.md §22) for rb_cql_grad / rb_cql_dueling_grad, with a derived
per-element error bound for the kernels' fp32 arithmetic.

For copy j of sample i (row r = jB + i of the online rows of s) with logits q_a [Z] and values Q_a (the expected value
over the support, or with no support the mean quantile):
  R_r = logsumexp_a Q_a - Q_{a_i},   sigma = softmax_a Q,   c = alpha w_i / (M B);
  g_ak = c (sigma_a - [a = a_i]) p_ak (z_k - Q_a)   (categorical),   c (sigma_a - [a = a_i]) / N   (quantile);
  gap_i = (1/M) sum_j R_r.  On the fused head dv_k = sum_a g_ak and dA_ak = g_ak - dv_k / A.

The bound follows the kernel's operation order with u = 2^-24 (each rounded op at most u relative; expf / logf a few
ulps, counted as 4u): the dueling combination x = v + adv - mean (e_x = 3u(|v| + |adv| + |mean|) + A u |mean|), then
  p:      |dp| <= p eps_p,        eps_p = 2 max e_x + (Z/32 + 12) u
  Q:      |dQ| <= eps_Q = S (eps_p + (Z/32 + 8) u),  S = sum p |z|      (quantile: e_x,max + (N/32 + 4) u sum|q| / N)
  sigma:  |dsigma_a| <= sigma_a eps_s,  eps_s = 2 max_a eps_Q,a + (A + 12) u
  c_a:    |dc_a| <= |c| (sigma_a eps_s + 6 u |sigma_a - d_a|)
  g:      |dg| <= |dc_a| |dq| + |c_a| p (eps_p |z - Q| + eps_Q,a + 3 u |z - Q|) + u |g|   (quantile: |dc_a| / N + u |g|)
then the dueling map (A u sum |g| for the value sum) and the final add (u |dz0 + g|).  The whole is doubled for the
second-order terms.  R: eps_Q,act + max eps_Q + (A + 12) u (|log S| + 1) + u |R|."""
import numpy as np
import torch

U = 2.0 ** -24
SAFETY = 2.0


def f32(x):
    return float(np.float32(x))


def _d(t):
    return t.detach().to("cpu", torch.float64)


def make_inputs(entry, B, A, Z, M, head, seed, alpha=0.7, support="pm10"):
    """Seeded fp32 inputs: rows (z rows [M B][Z + A Z] for "dueling", logits [M B][A][Z] for "plain"), actions [B],
    weights [B] in (0, 1], the support (None for head "quantile") and alpha."""
    g = torch.Generator().manual_seed(seed)
    n = M * B
    if entry == "dueling":
        rows = torch.randn(n, Z + A * Z, generator=g) * 1.5
    else:
        rows = torch.randn(n, A, Z, generator=g) * 1.5
    if head == "quantile":
        rows = rows * 4.0
        sup = None
    else:
        lo, hi = {"pm10": (-10.0, 10.0), "0to20": (0.0, 20.0), "pm1": (-1.0, 1.0)}[support]
        sup = torch.linspace(lo, hi, Z)
    actions = torch.randint(0, A, (B,), generator=g)
    weights = torch.rand(B, generator=g) * 0.9 + 0.1
    return dict(entry=entry, B=B, A=A, Z=Z, M=M, rows=rows.float(), actions=actions, weights=weights.float(),
                support=None if sup is None else sup.float(), alpha=f32(alpha))


def logits(inp):
    """(q [M B][A][Z] float64, e_x [M B][A][Z]): the rows the kernel forms, and the fp32 combination's error bound."""
    A, Z = inp["A"], inp["Z"]
    rows = _d(inp["rows"])
    if inp["entry"] != "dueling":
        return rows, torch.zeros_like(rows)
    v, adv = rows[:, :Z].unsqueeze(1), rows[:, Z:].view(-1, A, Z)
    mean = adv.mean(1, keepdim=True)
    ex = 3 * U * (v.abs() + adv.abs() + mean.abs()) + A * U * adv.abs().mean(1, keepdim=True)
    return v + adv - mean, ex.expand(-1, A, Z)


def values(q, support):
    """(Q [R][A], p [R][A][Z] or None) in float64."""
    if support is None:
        return q.mean(2), None
    p = torch.softmax(q, 2)
    return (p * support.view(1, 1, -1)).sum(2), p


def objective(q, actions, weights, support, alpha, M):
    """alpha (1 / (M B)) sum_ij w_i R_ij, differentiable in q [M B][A][Z]; and R [M B]."""
    B = actions.shape[0]
    Q, _ = values(q, support)
    act, w = actions.repeat(M), weights.double().repeat(M)
    R = torch.logsumexp(Q, 1) - Q[torch.arange(q.shape[0]), act]
    return alpha * (w * R).sum() / (M * B), R


def grad_logits(q, actions, weights, support, alpha, M):
    """(g [M B][A][Z], R [M B], sigma [M B][A], Q, p) in closed form."""
    B, (MB, A, Z) = actions.shape[0], q.shape
    Q, p = values(q, support)
    act, w = actions.repeat(M), weights.double().repeat(M)
    sigma = torch.softmax(Q, 1)
    R = torch.logsumexp(Q, 1) - Q[torch.arange(MB), act]
    d = sigma - torch.nn.functional.one_hot(act, A).double()
    ca = (alpha * w / (M * B)).unsqueeze(1) * d
    if support is None:
        g = (ca / Z).unsqueeze(2).expand(MB, A, Z).clone()
    else:
        g = ca.unsqueeze(2) * p * (support.view(1, 1, -1) - Q.unsqueeze(2))
    return g, R, sigma, Q, p


def dueling_map(g):
    """[M B][A][Z] logit gradients -> [M B][Z + A Z] (dv, dA) through the dueling combination."""
    dv = g.sum(1)
    return torch.cat([dv, (g - dv.unsqueeze(1) / g.shape[1]).flatten(1)], 1)


def reference(inp, dz0=None):
    """(out, e_out, gap, e_gap): the entry's output (dz0 + the mapped gradient, dz0 float64 of the incoming fp32
    gradient, zeros when None) and the gap [B], each with its per-element bound."""
    A, Z, M, B = inp["A"], inp["Z"], inp["M"], inp["B"]
    sup = None if inp["support"] is None else _d(inp["support"])
    q, ex = logits(inp)
    alpha = inp["alpha"]
    g, R, sigma, Q, p = grad_logits(q, inp["actions"], inp["weights"], sup, alpha, M)
    act = inp["actions"].repeat(M)
    w = _d(inp["weights"]).repeat(M)
    c = (alpha * w / (M * B)).unsqueeze(1)
    d = sigma - torch.nn.functional.one_hot(act, A).double()
    exm = ex.amax(2)                                            # [MB][A]
    if sup is None:
        eQ = exm + (Z / 32 + 4) * U * q.abs().mean(2)
    else:
        eps_p = (2 * exm + (Z / 32 + 12) * U).unsqueeze(2)
        S = (p * sup.abs().view(1, 1, -1)).sum(2)
        eQ = S * (eps_p.squeeze(2) + (Z / 32 + 8) * U)
    eps_s = (2 * eQ.amax(1) + (A + 12) * U).unsqueeze(1)
    dca = c.abs() * (sigma * eps_s + 6 * U * d.abs())
    ca = c * d
    if sup is None:
        eg = (dca / Z).unsqueeze(2).expand(-1, -1, Z) + U * g.abs()
    else:
        zq = (sup.view(1, 1, -1) - Q.unsqueeze(2)).abs()
        dq = p * zq
        eg = dca.unsqueeze(2) * dq + ca.abs().unsqueeze(2) * p * (eps_p * zq + eQ.unsqueeze(2) + 3 * U * zq) + U * g.abs()
    if inp["entry"] == "dueling":
        out = dueling_map(g)
        edv = eg.sum(1) + A * U * g.abs().sum(1)
        eda = eg + (edv + 2 * U * g.sum(1).abs()).unsqueeze(1) / A + U * (g.abs() + g.sum(1).abs().unsqueeze(1) / A)
        e_out = torch.cat([edv, eda.flatten(1)], 1)
    else:
        out, e_out = g, eg
    if dz0 is not None:
        out = out + _d(dz0).view_as(out)
    e_out = SAFETY * (e_out + U * out.abs())
    m = Q.amax(1)
    lse = torch.log(torch.exp(Q - m.unsqueeze(1)).sum(1))
    eR = eQ[torch.arange(M * B), act] + eQ.amax(1) + (A + 12) * U * (lse.abs() + 1) + U * R.abs()
    gap = R.view(M, B).mean(0)
    e_gap = SAFETY * (eR.view(M, B).sum(0) / M + M * U * gap.abs())
    return out, e_out, gap, e_gap


def emulate(inp, dz0=None):
    """The kernel's stated operation order in numpy fp32 (expf / logf by numpy's float32 exp / log): (out, gap)."""
    f = np.float32
    A, Z, M, B = inp["A"], inp["Z"], inp["M"], inp["B"]
    rows = inp["rows"].numpy().astype(f)
    sup = None if inp["support"] is None else inp["support"].numpy().astype(f)
    acts, w = inp["actions"].numpy(), inp["weights"].numpy().astype(f)
    alpha = f(inp["alpha"])
    out = np.zeros((M * B,) + rows.shape[1:], f) if dz0 is None else dz0.numpy().astype(f).reshape(rows.shape).copy()
    gap = np.zeros(B, f)
    for i in range(B):
        c = f(f(alpha * w[i]) / f(M * B))
        acc = f(0)
        for j in range(M):
            r = j * B + i
            if inp["entry"] == "dueling":
                v, adv = rows[r, :Z], rows[r, Z:].reshape(A, Z)
                mean = np.zeros(Z, f)
                for a in range(A):
                    mean = (mean + adv[a]).astype(f)
                mean = (mean / f(A)).astype(f)
                x = ((v + adv).astype(f) - mean).astype(f)
            else:
                x = rows[r]
            Q = np.zeros(A, f)
            dq = np.zeros((A, Z), f)
            for a in range(A):
                if sup is None:
                    Q[a] = f(np.sum(x[a], dtype=f) / f(Z))
                else:
                    e = np.exp((x[a] - x[a].max()).astype(f)).astype(f)
                    s = np.sum(e, dtype=f)
                    Q[a] = f(np.sum((sup * e).astype(f), dtype=f) / s)
                    dq[a] = ((e / s).astype(f) * (sup - Q[a]).astype(f)).astype(f)
            m = Q.max()
            S = f(0)
            for a in range(A):
                S = f(S + np.exp(f(Q[a] - m)))
            Rv = f(f(0) - f(f(Q[acts[i]] - m) - f(np.log(S))))
            acc = Rv if j == 0 else f(acc + Rv)
            pi = (np.exp((Q - m).astype(f)).astype(f) / S).astype(f)
            ca = (c * (pi - (np.arange(A) == acts[i]).astype(f)).astype(f)).astype(f)
            g = np.broadcast_to((ca / f(Z)).astype(f)[:, None], (A, Z)) if sup is None else (ca[:, None] * dq).astype(f)
            if inp["entry"] == "dueling":
                gv = np.zeros(Z, f)
                for a in range(A):
                    gv = (gv + g[a]).astype(f)
                da = (g - (gv * f(1.0 / A)).astype(f)).astype(f)
                out[r] = (out[r] + np.concatenate([gv, da.reshape(-1)])).astype(f)
            else:
                out[r] = (out[r] + g).astype(f)
        gap[i] = f(acc / f(M))
    return out, gap
