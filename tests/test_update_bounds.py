"""The bound of the whole-update comparison (update_ref.TAU_G) and the case table of tests/test_gpu_update_f64.py, on the
CPU.

TAU_G is the per-element bound |g - g64| <= TAU_G * scale of every gradient the learner's update computes, scale being
update_ref's absolute-value backward.  As for the stage bounds (tests/test_conv_bounds.py, tests/test_c51_adam_bounds.py)
it sits between two measurements:
  * at least 5x above the largest |err| / scale of the same update chain in fp32 (torch on the CPU: fp32 conv body, noisy
    dueling head, C51 projection / quantile loss and autograd) against update_ref in float64, on small nets at the
    table's shapes -- the error of an update done right;
  * at least 5x below the largest |err| / scale of each modelled wiring slip: gamma^n of the neighbouring horizon step,
    one sample's importance weight dropped, DrQ's loss over M B instead of B, the gradient taken with another noise draw
    -- what an update done wrong shows.
TAU_LOSS, the per-sample loss's bound relative to its scale (where the loss is beyond the north-star 1e-5), sits the same
way between the fp32 chain and gamma^n of the neighbouring horizon step.  The H100's observed ratios, per parameter group,
are in DESIGN.md §4."""
import argparse

import numpy as np
import pytest
import torch

import horizon_ref as HR
import update_cases as UC
import update_ref as U

A = 6


def make_args(**kw):
    d = dict(device=torch.device("cpu"), history_length=4, discount=0.99, multi_step=3, priority_weight=0.4,
             priority_exponent=0.5, atoms=51, V_min=-10.0, V_max=10.0, batch_size=32, norm_clip=10.0, model=None,
             learning_rate=6.25e-5, adam_eps=1.5e-4, architecture="canonical", hidden_size=64, noisy_std=0.1)
    d.update(kw)
    return argparse.Namespace(**d)


# ---- the case table -------------------------------------------------------------------------------------------------------
def test_table_covers_every_allowed_pair():
    assert UC.missing_pairs(UC.CASES) == []
    assert not any(UC.refused(c) for c in UC.CASES)
    assert [c["batch"] for c in UC.CASES].count(512) == 1
    assert 16 <= len(UC.CASES) <= 20
    assert len({UC.case_id(c) for c in UC.CASES}) == len(UC.CASES)


def test_left_out_pairs_are_refused():
    """QR x DrQ's copies is refused when the agent reads its arguments (DrQ on the library head is refused by learn()
    before it samples: test_gpu_drq.py::test_refusals)."""
    from rainbow_b200.agent import distribution_options
    for c in UC.CASES:
        distribution_options(make_args(**{k: v for k, v in UC.agent_kwargs(c).items()
                                          if k in ("distribution", "quantile_kappa", "augment_m", "augment_k")}))
    with pytest.raises(ValueError, match="augment_m"):
        distribution_options(make_args(distribution="quantile", augment_m=2, augment_k=2))
    assert UC.refused(dict(dist="quantile", aug="drq")) and UC.refused(dict(aug="drq", head="library"))


# ---- the fp32 chain ------------------------------------------------------------------------------------------------------
def _scaled(x):
    return x.sign() * x.abs().sqrt()


def _problem(arch, hidden, B, dist, M, K, seed):
    from rainbow_b200.model import DQN
    torch.manual_seed(seed)
    kw = dict(architecture=arch, hidden_size=hidden)
    if dist == "quantile":
        kw.update(distribution="quantile", atoms=32)
    net, tnet = DQN(make_args(**kw), A), DQN(make_args(**kw), A)
    net.train()
    tnet.train()
    P = {n: p.detach().clone() for n, p in net.named_parameters()}
    T = {n: (p.detach() + 0.01 * torch.randn_like(p)).clone() for n, p in net.named_parameters()}   # a target near it
    f = {n: (_scaled(torch.randn(m.in_features)), _scaled(torch.randn(m.out_features)))
         for n, m in net.named_children() if n.startswith("fc_")}
    rs = np.random.RandomState(seed)
    x = torch.from_numpy((rs.randint(0, 256, ((M + K) * B, 4, 84, 84)) / 255.0).astype(np.float32))
    nt = (rs.uniform(size=B) > 0.2).astype(np.float32)
    batch = dict(actions=torch.from_numpy(rs.randint(0, A, B)), returns=torch.from_numpy(rs.randint(-2, 3, B).astype(np.float32)),
                 nonterminals=torch.from_numpy(nt).view(B, 1), weights=torch.from_numpy(rs.uniform(0.3, 1.0, B).astype(np.float32)),
                 gamma_n=0.99 ** 3)
    if dist == "quantile":
        batch.update(kappa=1.0)
    else:
        batch.update(support=torch.linspace(-10.0, 10.0, 51), vmin=-10.0, vmax=10.0, dz=20.0 / 50)
    return net, tnet, P, T, f, x, batch


def _fp32_update(net, tnet, P, T, f, x, batch, dist, M, K):
    """The update in fp32 (torch, CPU): (loss [B], {name: gradient}, (conv sides, hidden sides), its online s' logits and
    their rounding scale (0: the arg-max reads them as they are))."""
    Pf = {n: t.clone().requires_grad_() for n, t in P.items()}
    keep, hidden = [], []
    q_on = _net32(net, Pf, f, x, keep, hidden)
    with torch.no_grad():
        q_t = _net32(tnet, T, f, x[M * x.shape[0] // (M + K):], [], [])
    B = q_t.shape[0] // K
    rows = torch.arange(B)
    r, nt, w = batch["returns"], batch["nonterminals"].view(-1), batch["weights"]
    gn = torch.tensor(np.float32(batch["gamma_n"]))
    targets = []
    with torch.no_grad():
        for k in range(K):
            q_ns = q_on[(M + k) * B:(M + k + 1) * B]
            if dist == "quantile":
                best = q_ns.mean(2).argmax(1)
                targets.append(r.unsqueeze(1) + (nt * gn).unsqueeze(1) * q_t[k * B:(k + 1) * B][rows, best])
                continue
            sup = batch["support"]
            best = (torch.softmax(q_ns, 2) * sup).sum(2).argmax(1)
            pt = torch.softmax(q_t[k * B:(k + 1) * B][rows, best], 1)
            Z = sup.numel()
            b = ((r.unsqueeze(1) + (nt * gn).unsqueeze(1) * sup).clamp(batch["vmin"], batch["vmax"]) - batch["vmin"]) / \
                torch.tensor(np.float32(batch["dz"]))
            lo, up = b.floor(), b.ceil()
            lo = torch.where((up > 0) & (lo == up), lo - 1, lo)
            up = torch.where((lo < Z - 1) & (lo == up), up + 1, up)
            m = torch.zeros(B, Z + 1)
            m.scatter_add_(1, lo.long(), pt * (up - b))
            m.scatter_add_(1, up.long(), pt * (b - lo))
            targets.append(m[:, :Z])
        tgt = sum(targets) / K
    loss = 0.0
    for j in range(M):
        qs = q_on[j * B:(j + 1) * B][rows, batch["actions"]]
        if dist == "quantile":
            N = qs.shape[1]
            u = tgt.unsqueeze(1) - qs.unsqueeze(2)
            tau = (2.0 * torch.arange(N, dtype=torch.float32) + 1.0) / (2.0 * N)
            tw = torch.where(u.detach() < 0, 1.0 - tau.view(1, N, 1), tau.view(1, N, 1))
            H = torch.where(u.abs() <= 1.0, 0.5 * u * u, u.abs() - 0.5)
            loss = loss + (tw * H).sum((1, 2)) / N
        else:
            loss = loss - (tgt * torch.log_softmax(qs, 1)).sum(1)
    loss = loss / M
    ((w * loss).sum() / B).backward()
    q_ns = q_on[M * B:].detach().double()
    return loss.detach(), {n: t.grad for n, t in Pf.items()}, ([(a > 0).double() for a in keep],
                                                              [(h > 0).double() for h in hidden]), (q_ns, torch.zeros_like(q_ns))


def _net32(net, P, f, x, keep, hidden):
    for m, (wn, bn) in zip(net.conv_layers(), U.conv_names(net)):
        x = torch.relu(torch.nn.functional.conv2d(x, P[wn], P[bn], m.stride, m.padding))
        keep.append(x.detach())
    x = x.reshape(x.shape[0], -1)

    def noisy(name, v):
        fi, fo = f[name]
        return torch.nn.functional.linear(v, P[f"{name}.weight_mu"] + P[f"{name}.weight_sigma"] * torch.outer(fo, fi),
                                          P[f"{name}.bias_mu"] + P[f"{name}.bias_sigma"] * fo)

    def hid(name):
        h = noisy(name, x)
        hidden.append(h.detach())
        return torch.relu(h)

    Z = net.atoms
    v = noisy("fc_z_v", hid("fc_h_v")).view(-1, 1, Z)
    a = noisy("fc_z_a", hid("fc_h_a")).view(-1, A, Z)
    return v + a - a.mean(1, keepdim=True)


def _ratios(grads, ref):
    return {n: U.ratio(g, ref["grads"][n], ref["scales"][n]) for n, g in grads.items()}


# the table's shapes on small nets: batch 1 / 32 / 33, canonical and data-efficient, both losses, DrQ's copies
SHAPES = [("canonical", 64, 32, "categorical", 1, 1), ("data-efficient", 64, 33, "quantile", 1, 1),
          ("canonical", 64, 8, "categorical", 2, 2), ("data-efficient", 256, 1, "categorical", 1, 1),
          ("canonical", 64, 33, "quantile", 1, 1)]


@pytest.mark.parametrize("shape", SHAPES, ids=[f"{s[0]}-h{s[1]}-B{s[2]}-{s[3]}-M{s[4]}K{s[5]}" for s in SHAPES])
def test_tau_g_is_5x_above_the_fp32_chain(shape):
    arch, hidden, B, dist, M, K = shape
    net, tnet, P, T, f, x, batch = _problem(arch, hidden, B, dist, M, K, seed=B + hidden)
    loss32, g32, sides, own = _fp32_update(net, tnet, P, T, f, x, batch, dist, M, K)
    ref = U.update_ref(net, P, f, x, sides, tnet, T, f, x[M * B:], batch, dist, M, K, own_ns=own)
    assert not ref["ties"], "no near-tied arg-max in these draws: the alternatives are not needed to pass"
    rl = float(((loss32.double() - ref["loss"]).abs() / ref["lscale"]).max())
    r = _ratios(g32, ref)
    worst = max(r, key=r.get)
    print(f"\n{shape}: largest |err| / scale {r[worst]:.3g} ({worst}); loss {rl:.3g} of its scale")
    assert 5 * r[worst] <= U.TAU_G, (worst, r[worst])
    assert 5 * rl <= U.TAU_LOSS, rl


def _slip_ratio(ref, slipped):
    return max(_ratios(slipped["grads"], ref).values())


@pytest.mark.parametrize("shape", SHAPES[:3], ids=[f"{s[0]}-B{s[2]}-{s[3]}-M{s[4]}" for s in SHAPES[:3]])
def test_tau_g_is_5x_below_the_modelled_slips(shape):
    arch, hidden, B, dist, M, K = shape
    net, tnet, P, T, f, x, batch = _problem(arch, hidden, B, dist, M, K, seed=B + hidden)
    _, _, sides, _ = _fp32_update(net, tnet, P, T, f, x, batch, dist, M, K)
    run = lambda b=batch, ff=f: U.update_ref(net, P, ff, x, sides, tnet, T, f, x[M * B:], b, dist, M, K)
    ref = run()
    slips = {}
    # the annealed horizon's nonterminals in discount form, fl32(nt gamma_u^n_u) with gamma_n = 1, at the previous step
    a = UC.ANNEAL
    steps = [HR.schedule(u, a["anneal_steps"], a["multi_step_start"], a["multi_step"], a["discount_start"], a["discount"])
             for u in (2, 3)]
    nt = batch["nonterminals"]
    disc = [dict(batch, gamma_n=1.0, nonterminals=(nt * np.float32(g ** n)).float()) for n, g in steps]
    at, prev = run(disc[1]), run(disc[0])
    slips["gamma^n of the neighbouring horizon step"] = _slip_ratio(at, prev)
    loss_slip = float(((prev["loss"] - at["loss"]).abs() / at["lscale"]).max())
    assert loss_slip >= 5 * U.TAU_LOSS, loss_slip
    w = batch["weights"].clone()
    w[B // 2] = 0.0
    slips["one sample's weight dropped"] = _slip_ratio(ref, run(dict(batch, weights=w)))
    if M > 1:
        slips["loss over M B"] = _slip_ratio(ref, dict(grads={n: g / M for n, g in ref["grads"].items()}))
    other = {n: (_scaled(torch.randn(fi.shape)), _scaled(torch.randn(fo.shape))) for n, (fi, fo) in f.items()}
    slips["gradient from another noise draw"] = _slip_ratio(ref, run(ff=other))
    print(f"\n{shape}: " + "; ".join(f"{k} {v:.3g}" for k, v in slips.items()) + f"; loss, neighbouring horizon {loss_slip:.3g}")
    for k, v in slips.items():
        assert v >= 5 * U.TAU_G, (k, v)


def test_near_tied_arg_max_gives_every_accepted_choice():
    """A row whose online s' logits tie exactly on two actions: the reference returns the update under each."""
    B, M, K = 4, 1, 1
    net, tnet, P, T, f, x, batch = _problem("data-efficient", 64, B, "categorical", M, K, seed=7)
    _, _, sides, (q, L) = _fp32_update(net, tnet, P, T, f, x, batch, "categorical", M, K)
    q = q.clone()
    q[0, 1] = q[0, 0]
    q[0, 2:] = 0.0
    q[0, 2:, 0] = 20.0                               # actions 0 and 1 tie; the rest put their mass on V_min
    ref = U.update_ref(net, P, f, x, sides, tnet, T, f, x[M * B:], batch, "categorical", M, K, own_ns=(q, L))
    assert [(k, i) for k, i, _ in ref["ties"]] == [(0, 0)] and sorted(ref["ties"][0][2]) == [0, 1]
    (alt,) = ref["alternatives"]
    assert {int(ref["astar"][0, 0]), int(alt["astar"][0, 0])} == {0, 1}
    assert torch.equal(ref["astar"][:, 1:], alt["astar"][:, 1:])
