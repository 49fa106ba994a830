"""Float64 reference of the distributional loss (csrc/rb_kernels.cu: k_c51 behind rb_c51_loss_grad, k_c51_dueling behind
rb_c51_dueling_loss_grad) with a condition scale for every output element, and the seeded inputs its tests draw.

As in tests/head_ref.py everything is computed from the SAME fp32 tensors the kernel reads, and each stage takes the
kernel's own result of the stage before it, so a wrong element is blamed on the stage that produced it:
  arg-max    the expected value of every action of online(s'), ev[a], with the scale of head_ref.expectation.  The
             kernel's a* is accepted if ev[a*] >= max_a ev - TAU_EV (scale[a*] + scale[argmax]) (both expected values
             are off by at most TAU_EV times their scale); rows that are bit-identical across actions must give the
             first one, exactly (tested by the caller).  Everything after it uses the kernel's a*.
  projection pt = softmax(target at a*), Tz = clamp(r + nt gamma^n s, Vmin, Vmax), b = (Tz - Vmin) / dz with the fp32 dz
             the kernel was passed, l = floor(b), u = ceil(b) and the reference's two fix-ups (agent.py:82-86).  When
             fp32 rounding puts b just past Z - 1 (Tz = Vmax at e.g. Z 62 with V +-1, or Z 100 with V +-100), u = Z: the
             kernel drops that contribution pt (b - l) (at most pt times the rounding of b), and so does this reference.
             The reference's index_add_ over the flattened batch adds it to atom 0 of the next sample instead (past the
             end of m for the last one).
  m          is continuous in b (at an integer b all of pt_j lands on atom b either way), so a per-element bound needs
             no special cases: scale_k = sum over the atoms j with |b_j - k| < 1 + RHO of
             pt_j (1 + c_j + (|r| + |nt gamma^n s_j| + |Vmin|) / dz), the last term being the rounding of b_j in units
             of u, c_j that of the logits (below).  RHO covers the rounding of b across an integer.
  loss, grad from the kernel's m: loss = -sum m log p, g = (w/B)(p sum m - m) of the online row of the taken action, with
             the scales sum |m| (1 + |log p| + c) and |w/B| (p (1 + c) sum |m| + |m|).  Dueling: dz_v = g,
             dz_a[a] = g ([a == act] - 1/A), scale that of g times |[a == act] - 1/A|.
c_j = Lf_j + sum_i p_i Lf_i bounds, in units of u, what the error of the fp32 logits does to log p_j and p_j:
Lf = L + |q - max q|, L the scale of the dueling combination (head_ref._dueling; 0 for the plain entry point, whose
logits are inputs) and |q - max q| the rounding of the kernel's x - max before expf.  Every scale also carries FLOOR, far
below any value that matters and far above fp32's underflow spacing (2^-149): a probability the kernel rounds to zero
(e^-150 of a sharp row) is then not an error.  The gradient's FLOOR is scaled by |w/B| so that weight 0 gives exact 0.

The bounds (TAU, TAU_EV) are derived in tests/test_c51_adam_bounds.py: at least 5x above the fp32 arithmetic of the same
operation (the CPU oracle, oracle/rb_oracle.c orc_c51), at least 5x below each semantic slip it tests."""
import numpy as np
import torch

import head_ref as R

TAU_EV = 1e-6           # the arg-max's expected values
TAU = 2e-6              # m, loss, grad / dz
RHO = 1e-3
FLOOR = 2.0 ** -100

SUPPORTS = {"pm10": (-10.0, 10.0), "0to20": (0.0, 20.0), "m3to7": (-3.0, 7.0), "pm1": (-1.0, 1.0), "pm100": (-100.0, 100.0),
            "rev": (-10.0, 10.0)}
GAMMA_N = 0.99 ** 3


def _d(t):
    return t.double()


def f32(v):
    return float(np.float32(v))


def support_of(kind, Z):
    """(support [Z] fp32, Vmin, Vmax, dz) the way the agent builds them (linspace, (Vmax - Vmin) / (Z - 1)); "rev" is the
    decreasing support, the one input that takes the projection's full-scan branch."""
    vmin, vmax = SUPPORTS[kind]
    s = torch.linspace(vmin, vmax, Z)
    if kind == "rev":
        s = s.flip(0).contiguous()
    return s, vmin, vmax, (vmax - vmin) / (Z - 1)


# row kinds, cycled over the batch (coprime periods, so every combination occurs in a batch of 35 or more)
RET_KINDS = ("spread", "terminal", "below", "above", "on_atom")    # period 5
LOGIT_KINDS = ("n2", "sharp", "const", "ties")                     # period 4
W_PERIOD = 7                                                       # weight 0 at i % 7 == 3, 1 at i % 7 == 5

# (B, A, Z, support) of the grid both entry points run (tests/test_gpu_c51_f64.py) and the oracle is measured on
# (tests/test_c51_adam_bounds.py): Z across the R = 2 / R = 4 switch at 64, A past the dueling kernel's 8 warps, B with
# k_c51's last CTA partly idle, the two supports whose b rounds past Z - 1 at Vmax (Z 62 V +-1, Z 100 V +-100)
CASES = [(32, 6, 51, "pm10"), (5, 2, 2, "pm10"), (3, 18, 3, "0to20"), (33, 6, 31, "m3to7"), (35, 1, 32, "pm10"),
         (1, 64, 33, "0to20"), (512, 6, 51, "pm10"), (33, 18, 64, "m3to7"), (5, 6, 65, "pm10"), (40, 2, 101, "0to20"),
         (3, 18, 128, "m3to7"), (35, 6, 62, "pm1"), (35, 6, 100, "pm100"), (35, 6, 51, "rev"), (5, 6, 128, "rev"),
         (2048, 6, 51, "pm10"), (1, 1, 128, "pm10"), (32, 64, 101, "0to20"), (35, 2, 128, "pm10")]


def make_inputs(entry, B, A, Z, sup_kind, seed):
    """Seeded fp32 inputs of one case (CPU tensors).  Returns per row i:
      returns / nonterminals by RET_KINDS[i % 5]: spread r in [Vmin - span/4, Vmax + span/4]; terminal (nt 0); below
        Vmin - gamma^n max|s| (every atom at b = 0: the second fix-up); above Vmax + gamma^n max|s| (every atom at
        b = Z - 1: the first fix-up); on_atom (nt 0, r an atom of the support: an interior integer b);
      logits by LOGIT_KINDS[i % 4]: N(0, 2), sharp N(0, 30), constant rows, or online(s') rows identical across actions
        (a tie: the first action must win);
      weights U(0.2, 1) with 0 and 1 rows.
    entry "plain": q_on_s, q_on_ns, q_tg_ns [B][A][Z]; entry "dueling": z_on [2B][Z + A Z] (s rows, then s'), z_tg [B][..]."""
    g = torch.Generator().manual_seed(seed)
    support, vmin, vmax, dz = support_of(sup_kind, Z)
    span, smax = vmax - vmin, max(abs(vmin), abs(vmax))
    rets, nts = torch.empty(B), torch.ones(B, 1)
    for i in range(B):
        kind = RET_KINDS[i % 5]
        u = float(torch.rand(1, generator=g))
        if kind == "spread":
            rets[i] = vmin - span / 4 + u * 1.5 * span
            nts[i] = float(u < 0.8)
        elif kind == "terminal":
            rets[i], nts[i] = vmin + u * span, 0.0
        elif kind == "below":
            rets[i] = vmin - GAMMA_N * smax - (0.01 + u) * span
        elif kind == "above":
            rets[i] = vmax + GAMMA_N * smax + (0.01 + u) * span
        else:
            rets[i], nts[i] = support[int(u * Z)], 0.0
    w = torch.rand(B, generator=g) * 0.8 + 0.2
    w[torch.arange(B) % W_PERIOD == 3] = 0.0
    w[torch.arange(B) % W_PERIOD == 5] = 1.0
    acts = torch.randint(0, A, (B,), generator=g)
    ncol = A * Z if entry == "plain" else Z + A * Z
    rows = {k: torch.randn(B, ncol, generator=g) for k in ("s", "ns", "t")}
    lk = torch.arange(B) % 4
    for k, t in rows.items():
        t[lk == 0] *= 2.0
        t[lk == 1] *= 30.0
        # constant rows: one value per logit row (plain) / per stream row (dueling)
        blocks = t[lk == 2].view(-1, ncol // Z, Z)
        t[lk == 2] = blocks[:, :, :1].expand_as(blocks).reshape(-1, ncol) * 2.0
        t[lk == 3] *= 2.0
    ns = rows["ns"][lk == 3]                                            # ties: online(s') identical across actions
    first = Z if entry == "dueling" else 0
    ns[:, first:] = ns[:, first:first + Z].repeat(1, A)
    rows["ns"][lk == 3] = ns
    inp = dict(entry=entry, B=B, A=A, Z=Z, support=support, vmin=vmin, vmax=vmax, dz=dz, gamma_n=GAMMA_N, actions=acts,
               returns=rets, nonterminals=nts, weights=w)
    if entry == "plain":
        inp.update(q_on_s=rows["s"].view(B, A, Z), q_on_ns=rows["ns"].view(B, A, Z), q_tg_ns=rows["t"].view(B, A, Z))
    else:
        inp.update(z_on=torch.cat([rows["s"], rows["ns"]]), z_tg=rows["t"])
    return inp


def to(inp, device):
    return {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in inp.items()}


def logits(inp, which):
    """(q [B][A][Z], L) in float64 of online(s) ("s"), online(s') ("ns") or target(s') ("t")."""
    B, A, Z = inp["B"], inp["A"], inp["Z"]
    if inp["entry"] == "plain":
        q = _d(inp[{"s": "q_on_s", "ns": "q_on_ns", "t": "q_tg_ns"}[which]])
        return q, torch.zeros_like(q)
    z = {"s": inp["z_on"][:B], "ns": inp["z_on"][B:], "t": inp["z_tg"]}[which]
    return R._dueling(z, A, Z)


def _softmax_terms(q, L):
    """p, log p, c (rows of the last dim) and Lf = L + |q - max q|."""
    lf = L + (q - q.max(-1, keepdim=True).values).abs()
    logp = torch.log_softmax(q, -1)
    p = logp.exp()
    return p, logp, lf + (p * lf).sum(-1, keepdim=True), lf


def expected_values(inp):
    """ev [B][A] of online(s') and its scale."""
    q, L = logits(inp, "ns")
    lf = L + (q - q.max(-1, keepdim=True).values).abs()
    return R.expectation(q, lf, inp["support"])


def _row(q, idx):
    return q[torch.arange(q.shape[0], device=q.device), idx.long()]


def projection(inp, astar):
    """m [B][Z] and its scale, for the kernel's a*."""
    Z = inp["Z"]
    q, L = logits(inp, "t")
    pt, _, c, _ = _softmax_terms(_row(q, astar), _row(L, astar))
    s = _d(inp["support"]).unsqueeze(0)
    r, nt = _d(inp["returns"]).unsqueeze(1), _d(inp["nonterminals"]).view(-1, 1)
    vmin, vmax, dz, gn = f32(inp["vmin"]), f32(inp["vmax"]), f32(inp["dz"]), f32(inp["gamma_n"])
    tz = (r + nt * gn * s).clamp(vmin, vmax)
    b = (tz - vmin) / dz
    lo, up = b.floor(), b.ceil()
    lo = torch.where((up > 0) & (lo == up), lo - 1, lo)
    up = torch.where((lo < Z - 1) & (lo == up), up + 1, up)
    m = torch.zeros(b.shape[0], Z + 1, dtype=torch.float64, device=b.device)      # column Z: the dropped contributions
    m.scatter_add_(1, lo.long(), pt * (up - b))
    m.scatter_add_(1, up.long(), pt * (b - lo))
    wj = pt * (1 + c + (r.abs() + (nt * gn * s).abs() + abs(vmin)) / dz)
    scale = torch.full((b.shape[0], Z), FLOOR, dtype=torch.float64, device=b.device)
    base = b.floor().long()
    for off in range(-2, 3):
        k = base + off
        near = ((k - b).abs() < 1 + RHO) & (k >= 0) & (k < Z)
        scale.scatter_add_(1, k.clamp(0, Z - 1), torch.where(near, wj, 0.0))
    return m[:, :Z], scale


def loss_grad(inp, m):
    """From the kernel's m [B][Z]: (loss, scale) [B] and (g, scale) [B][Z], the gradient row of the taken action."""
    q, L = logits(inp, "s")
    acts = inp["actions"]
    p, logp, c, _ = _softmax_terms(_row(q, acts), _row(L, acts))
    m = _d(m)
    loss = -(m * logp).sum(1)
    loss_scale = (m.abs() * (1 + logp.abs() + c)).sum(1) + FLOOR
    wi = (_d(inp["weights"]) / inp["B"]).unsqueeze(1)
    g = wi * (p * m.sum(1, keepdim=True) - m)
    g_scale = wi.abs() * (p * (1 + c) * m.abs().sum(1, keepdim=True) + m.abs() + FLOOR)
    return (loss, loss_scale), (g, g_scale)


def dueling_dz(inp, g, g_scale):
    """(dz, scale) [B][Z + A Z] of the dueling entry point from the gradient row g [B][Z] of the taken action."""
    B, A, Z = inp["B"], inp["A"], inp["Z"]
    sel = torch.zeros(B, A, 1, dtype=torch.float64, device=g.device)
    sel[torch.arange(B), inp["actions"].long()] = 1.0
    f = sel - 1.0 / A
    dza, sa = g.unsqueeze(1) * f, g_scale.unsqueeze(1) * f.abs()
    return torch.cat([g, dza.reshape(B, A * Z)], 1), torch.cat([g_scale, sa.reshape(B, A * Z)], 1)


def astar_ok(ev, scale, astar):
    """Rows whose a* is within the arg-max's rounding (see the module docstring)."""
    best = ev.argmax(1)
    slack = TAU_EV * (_row(scale, astar) + _row(scale, best))
    return _row(ev, astar) >= _row(ev, best) - slack


def first_of_identical(inp, astar):
    """Rows where no action before a* has an online(s') row bit-identical to a*'s (a tie must go to the first)."""
    B, A, Z = inp["B"], inp["A"], inp["Z"]
    if inp["entry"] == "plain":
        rows = inp["q_on_ns"]
    else:
        rows = inp["z_on"][B:, Z:].reshape(B, A, Z)            # zv and the mean are shared: equal za rows, equal logits
    same = (rows == _row(rows, astar).unsqueeze(1)).all(2)    # [B][A]
    before = torch.arange(A, device=rows.device).unsqueeze(0) < astar.long().unsqueeze(1)
    return ~(same & before).any(1)
