"""The learner under args.value_transform = "rescale" on the GPU, for both distributions.

* Agent.q_support is vt_ref's fl32(h^-1(support)) bitwise.
* One eager learn() per learner case (fused head pending / flushed, batch 64, C3, library head): flat_grad equals float64
  autograd of the transformed objective through float64 copies of both nets (§4's bounds), the losses equal its
  per-sample losses, and the sum-tree leaves are fl32(sqrt(loss)) of the kernel's losses.
* Five graph replays equal five eager updates bitwise; the update graph has the untransformed graph's launches with the
  loss kernel's value-rescaled instantiation in place of its sibling.
* value_transform "none" (and absent) gives the default agent: same graph, same results, bitwise.
* An annealed horizon equals the fixed one at each (n, gamma), bitwise.
* Acting / evaluate_q_memory return float64 return-unit Q on the fused and the library head; the statistics record's
  q_mean and target_mean are in return units.
* Checkpoints: resume equals never stopping; a checkpoint with the other transform or eps is refused without a write.
* Every compatible switch on at once: graph replays equal eager updates."""
import json
import re

import numpy as np
import pytest
import torch

import vt_ref as V
from helpers import assert_bits_equal
from conv_ref import conv_masks
from test_gpu_adamw import LEARNER_CASES
from test_gpu_augment import update_graph
from test_gpu_drq import TOL
from test_gpu_parity import DEV, FakeEnv, cpu, make_args, synthetic_ring
from update_ref import f64_forward, f64_forward_masked

pytestmark = pytest.mark.gpu

CAP = 8192
E3 = float(np.float32(1e-3))
VT = dict(value_transform="rescale")
DISTS = {"categorical": dict(), "quantile": dict(distribution="quantile", quantile_kappa=1.0)}
BBF = dict(anneal_steps=6, multi_step_start=10, discount_start=0.97, multi_step=3, discount=0.997)


@pytest.fixture(autouse=True)
def deterministic_cudnn():
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = old


def _agent(seed=5, **kw):
    from rainbow_b200.agent import Agent
    torch.manual_seed(seed)
    return Agent(make_args(**kw), FakeEnv(6))


def _memory(**args):
    mem, _ = synthetic_ring(CAP, seed=3, args=args)
    mem.seed = 99
    return mem


def _snapshot(ag, mem):
    torch.cuda.synchronize()
    o = ag.optimiser
    return {k: cpu(v).copy() for k, v in dict(tree=mem.transitions.tree, flat_param=o.flat_param, exp_avg=o.exp_avg,
                                               exp_avg_sq=o.exp_avg_sq, target=ag.target_flat).items()}


def _assert_snapshots(a, b, what):
    for k in a:
        assert_bits_equal(a[k], b[k], f"{k} {what}")


def _q_support_ref(ag):
    """s~ = fl32(h^-1(z_j)) of the agent's fp32 support, from vt_ref (not from the agent under test)."""
    return V.q_support(ag.support.cpu(), ag.value_transform_eps).to(DEV)


def _f64_objective(ag, q_s, q_ns, q_t, ws):
    """(per-sample loss, objective (1/B) sum_b w_b loss_b) of the transformed loss in float64, differentiable in q_s
    (logits / quantiles [B][A][Z] of online(s)); the arg-max and the target from the float64 online(s') and target(s')
    rows, s~ from vt_ref; nonterminals enter only as fl32(nt gamma_n), as in the kernels."""
    eps, B = ag.value_transform_eps, ws.B
    idx = torch.arange(B, device=DEV)
    with torch.no_grad():
        sc = (ws.nonterminals.view(-1).float() * np.float32(ag._gamma_n())).double().unsqueeze(1)
        r = ws.returns.double().view(-1, 1)
        if ag.quantile:
            astar = V.hinv(q_ns, eps).mean(2).argmax(1)
            T = V.h(r + sc * V.hinv(q_t[idx, astar], eps), eps)
        else:
            sq = _q_support_ref(ag).double()
            astar = (torch.softmax(q_ns, 2) * sq).sum(2).argmax(1)
            pt = torch.softmax(q_t[idx, astar], 1)
            Z = sq.numel()
            vmin, vmax, dz = (float(np.float32(v)) for v in (ag.Vmin, ag.Vmax, ag.delta_z))
            b = (V.h(r + sc * sq.unsqueeze(0), eps).clamp(vmin, vmax) - vmin) / dz
            lo, up = b.floor(), b.ceil()
            lo = torch.where((up > 0) & (lo == up), lo - 1, lo)
            up = torch.where((lo < Z - 1) & (lo == up), up + 1, up)
            m = torch.zeros(B, Z + 1, dtype=torch.float64, device=DEV)
            m.scatter_add_(1, lo.long(), pt * (up - b))
            m.scatter_add_(1, up.long(), pt * (b - lo))
            m = m[:, :Z]
    if ag.quantile:
        th = q_s[idx, ws.actions]
        N = th.shape[1]
        u = T.unsqueeze(1) - th.unsqueeze(2)
        tau = (torch.arange(N, dtype=torch.float64, device=DEV) + 0.5) / N
        tw = torch.where(u.detach() < 0, 1.0 - tau.view(1, N, 1), tau.view(1, N, 1))
        k = ag.quantile_kappa
        H = torch.where(u.abs() <= k, 0.5 * u * u, k * (u.abs() - 0.5 * k))
        loss = (tw * H).sum((1, 2)) / (N * k)
    else:
        loss = -(m * torch.log_softmax(q_s[idx, ws.actions], 1)).sum(1)
    return loss, (ws.weights.double().view(-1) * loss).sum() / B


@pytest.mark.parametrize("eps", [0.0, 1e-3, 1e-2])
@pytest.mark.parametrize("atoms,vmin,vmax", [(51, -10.0, 10.0), (2, -1.0, 3.0), (128, -20.0, 5.0)])
def test_q_support_is_the_reference(atoms, vmin, vmax, eps):
    """Agent.q_support, the one host-computed input the C51 kernels take under the transform, is vt_ref's s~ bitwise
    (and the support itself with the transform off)."""
    ag = _agent(atoms=atoms, V_min=vmin, V_max=vmax, value_transform="rescale", value_transform_eps=eps)
    ref = _q_support_ref(ag)
    assert ag.q_support.dtype == torch.float32 and torch.equal(ag.q_support, ref)
    assert not torch.equal(ref, ag.support), "the transform moves the support"
    off = _agent(atoms=atoms, V_min=vmin, V_max=vmax)
    assert off.q_support is off.support


@pytest.mark.parametrize("case", list(LEARNER_CASES))
@pytest.mark.parametrize("dist", list(DISTS))
def test_learner_gradient_is_f64_autograd(dist, case):
    """One eager learn() per case of test_gpu_adamw.LEARNER_CASES (fused head with the online draw pending / flushed,
    batch 64, C3, the library head): flat_grad equals float64 autograd of the transformed objective through float64
    copies of both nets on the update's own batch, noise factors and conv ReLU sides (§4's bounds), the losses equal its
    per-sample losses, and the sum-tree leaves are fl32(sqrt(loss)) of the kernel's losses, bitwise."""
    kw, pending = LEARNER_CASES[case]
    ag, mem = _agent(cuda_graph=False, **VT, **DISTS[dist], **kw), _memory()
    assert ag.value_transform_eps == E3
    on, tg, opt = ag.online_net, ag.target_net, ag.optimiser
    assert ag._fused_path(ag.batch_size) == (case != "library-head") and mem.priority_exponent == 0.5
    for step in range(2):
        ag.reset_noise()
        if not pending:
            on.flush_noise()
        torch.cuda.synchronize()
        P = {n: p.detach().double().requires_grad_() for n, p in on.named_parameters()}
        T = {n: p.detach().double() for n, p in tg.named_parameters()}
        p_before = opt.flat_param.clone()
        ag.learn(mem)
        torch.cuda.synchronize()
        ws = mem._last
        B = ws.B
        masks = conv_masks(ag, ws, p_before)
        q_on = f64_forward_masked(on, P, on.noise_factors(), ws.both_states.double(), masks)
        with torch.no_grad():
            q_t = f64_forward(tg, T, tg.noise_factors(), ws.next_states.double())
        loss, obj = _f64_objective(ag, q_on[:B], q_on[B:].detach(), q_t, ws)
        obj.backward()
        got = ag.last_loss.double()
        assert float(((got - loss.detach()).abs() / (loss.detach().abs() + 1.0)).max()) <= TOL["loss"], \
            f"loss, update {step}"
        tidx, l32 = cpu(ws.tree_idx), cpu(ag.last_loss)
        last = np.array([i for i in range(len(tidx)) if tidx[i] not in tidx[i + 1:]])   # duplicates: the last write wins
        assert_bits_equal(cpu(mem.transitions.tree)[tidx[last]], np.sqrt(l32)[last], f"priorities, update {step}")
        for n, p in on.named_parameters():
            off = (p.data_ptr() - opt.flat_param.data_ptr()) // 4
            d = float((opt.flat_grad[off:off + p.numel()].double() - P[n].grad.reshape(-1)).abs().max())
            tol = TOL["grad_conv" if n.startswith("convs") else "grad_head"]
            assert d <= tol, f"gradient of {n}, update {step}: {d:.3g}"


@pytest.mark.parametrize("dist", list(DISTS))
def test_graph_replays_equal_eager_updates(dist):
    kw = dict(VT, **DISTS[dist])
    ga, ea = _agent(**kw), _agent(cuda_graph=False, **kw)
    gm, em = _memory(), _memory()
    for step in range(7):
        for ag, mem in ((ga, gm), (ea, em)):
            ag.reset_noise()
            ag.learn(mem)
        assert_bits_equal(cpu(ga.last_loss), cpu(ea.last_loss), f"loss of update {step}")
        _assert_snapshots(_snapshot(ga, gm), _snapshot(ea, em), f"after update {step}")
    assert ga._graphs and not ea._graphs


@pytest.mark.parametrize("dist", list(DISTS))
def test_update_graph_swaps_only_the_loss_instantiation(dist, tmp_path, monkeypatch):
    names = {}
    for tag, kw in (("default", dict()), ("none", dict(value_transform="none")), ("vt", VT)):
        names[tag] = update_graph(_agent(**kw, **DISTS[dist]), _memory(), tmp_path / f"{tag}.dot", monkeypatch)
    assert names["none"] == names["default"], "value_transform 'none' leaves the update graph as it is"
    assert names["vt"] == names["default"], "the same launches (kernel nodes by name, template arguments aside)"
    loss = "k_qr_dueling" if dist == "quantile" else "k_c51_dueling"
    for tag, flag in (("default", "Lb0E"), ("vt", "Lb1E")):
        dot = open(tmp_path / f"{tag}.dot").read()
        assert re.search(rf"{len(loss)}{loss}ILi[24]E{flag}E", dot), f"{tag}: {loss}<R, {flag == 'Lb1E'}> launched"


@pytest.mark.parametrize("dist", list(DISTS))
def test_none_equals_the_default_bitwise(dist):
    a, b = _agent(cuda_graph=False, **DISTS[dist]), _agent(cuda_graph=False, value_transform="none", **DISTS[dist])
    ma, mb = _memory(), _memory()
    assert b.value_transform is None and b.q_support is b.support
    for step in range(3):
        for ag, mem in ((a, ma), (b, mb)):
            ag.reset_noise()
            ag.learn(mem)
        _assert_snapshots(_snapshot(a, ma), _snapshot(b, mb), f"after update {step}")


@pytest.mark.parametrize("dist", list(DISTS))
def test_annealed_horizon_equals_fixed(dist):
    """Each annealed update equals the fixed-horizon update at its (n, gamma) on the same rows and noise, bitwise: the
    transformed targets see s only as fl32(nonterminal gamma_n), like the untransformed ones (§12)."""
    from test_gpu_horizon import Out, lib, p, stream
    kw = dict(VT, **DISTS[dist])
    ag, plain = _agent(cuda_graph=False, **kw, **BBF), _agent(cuda_graph=False, **kw)
    mem = _memory(**BBF)
    seen = set()
    for u in range(8):
        n_u, g_u = ag.horizon()
        seen.add(n_u)
        for a in (ag, plain):
            a.reset_noise()
        ag.learn(mem)
        ws = mem._last
        B = ws.B
        gp = torch.tensor([g_u ** k for k in range(n_u)], dtype=torch.float32, device=DEV)
        out = Out(B, 4)
        tr = mem.transitions
        assert lib().rb_gather(p(tr.frames), p(tr.timestep), p(tr.action), p(tr.reward), p(tr.nonterminal), tr.size,
                               p(ws.data_idx), B, 4, n_u, p(gp), p(out.states), p(out.next_states), p(out.actions),
                               p(out.returns), p(out.nonterminals), stream()) == 0
        both = torch.cat([out.states, out.next_states])
        batch = (ws.tree_idx.clone(), both[:B], out.actions, out.returns, both[B:], out.nonterminals.view(B, 1),
                 ws.weights.clone())
        plain.n, plain.discount = n_u, g_u
        loss = plain._update_from_batch(batch, gate=ws.status)
        torch.cuda.synchronize()
        assert_bits_equal(cpu(ag.last_loss), cpu(loss), f"loss of update {u}")
        for name in ("flat_param", "exp_avg", "exp_avg_sq"):
            assert_bits_equal(cpu(getattr(ag.optimiser, name)), cpu(getattr(plain.optimiser, name)), f"{name} after {u}")
    assert len(seen) >= 4


@pytest.mark.parametrize("head", ["fused", "library"])
@pytest.mark.parametrize("dist", list(DISTS))
def test_acting_in_return_units(dist, head):
    """act / evaluate_q_memory / q_select against float64 return-unit Q of the eval-mode net: rb_q_values over s~ or
    rb_qr_vt_q_values on the fused head, the torch float32 fallback on the library head."""
    ag = _agent(architecture="data-efficient", hidden_size=64, **VT, **DISTS[dist])
    ag.eval()
    ag.online_net.use_fused_head = head == "fused"
    eps = ag.value_transform_eps
    val, _ = synthetic_ring(256, seed=4)
    on = ag.online_net
    with torch.no_grad():
        states = val.iter_states(0, val.capacity)
        P = {n: p.detach().double() for n, p in on.named_parameters()}
        f = {n: (torch.zeros(m.in_features, device=DEV), torch.zeros(m.out_features, device=DEV))
             for n, m in on.named_children() if n.startswith("fc_")}
        q = f64_forward(on, P, f, states.double())
        q = V.hinv(q, eps).mean(2) if ag.quantile else (torch.softmax(q, 2) * _q_support_ref(ag).double()).sum(2)
    assert ag.online_net.fused_ok(val.capacity) == (head == "fused")
    best_v, best_a = q.max(1)
    values = torch.tensor(ag.evaluate_q_memory(val), dtype=torch.float64, device=DEV)
    assert float((values - best_v).abs().max()) <= 1e-5 * float(best_v.abs().max() + 1)
    a, v = ag.q_select(states)
    gap = q.topk(2, 1).values
    clear = (gap[:, 0] - gap[:, 1]) > 1e-5 * (gap[:, 0].abs() + 1)
    assert torch.equal(a[clear], best_a[clear])
    for i in range(3):
        if bool(clear[i]):
            assert ag.act(states[i]) == int(best_a[i])


@pytest.mark.parametrize("dist", list(DISTS))
def test_statistics_in_return_units(dist):
    ag, mem = _agent(cuda_graph=False, learn_stats=8, **VT, **DISTS[dist]), _memory()
    eps = ag.value_transform_eps
    for _ in range(2):
        ag.reset_noise()
        ag.learn(mem)
    torch.cuda.synchronize()
    rec, last, B = ag.learn_stats(), ag._stats["last"], mem._last.B
    A, Z = ag.action_space, ag.atoms
    z = last["z"][:B].double()                 # the fused head's online(s) rows of the update
    q = z[:, :Z].unsqueeze(1) + z[:, Z:].view(B, A, Z) - z[:, Z:].view(B, A, Z).mean(1, keepdim=True)
    q = q[torch.arange(B, device=DEV), mem._last.actions]
    if ag.quantile:
        tm = float(V.hinv(last["m"].double(), eps).mean())
        qm = float(V.hinv(q, eps).mean())
    else:
        sq = _q_support_ref(ag).double()
        tm = float((last["m"].double() * sq).sum(1).mean())
        qm = float((torch.softmax(q, 1) * sq).sum(1).mean())
    assert rec["target_mean"][-1] == pytest.approx(tm, rel=1e-5, abs=1e-5)
    assert rec["q_mean"][-1] == pytest.approx(qm, rel=1e-5, abs=1e-5)


def test_resume_equals_never_stopping(tmp_path):
    from test_gpu_checkpoint import _agent as ck_agent
    from test_gpu_checkpoint import _assert_same, _before_update, _fresh_memory, _state, _update
    from test_gpu_checkpoint import _memory as ck_memory
    kw = dict(VT, value_transform_eps=1e-2)
    total, save_at = 10, 4
    ag, mem = ck_agent(**kw), ck_memory()
    losses = []
    for step in range(total):
        _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    run_a = _state(ag, mem, losses)
    ag, mem = ck_agent(**kw), ck_memory()
    losses = []
    for step in range(save_at):
        _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _before_update(ag, mem, save_at, True)
    ag.save_checkpoint(str(tmp_path / "ck"), mem)
    hp = json.load(open(tmp_path / "ck" / "rank0" / "manifest.json"))["hyper_parameters"]
    assert (hp["value_transform"], hp["value_transform_eps"]) == ("rescale", float(np.float32(1e-2)))
    ag, mem = ck_agent(seed=77, **kw), _fresh_memory()
    ag.load_checkpoint(str(tmp_path / "ck"), mem)
    for step in range(save_at, total):
        if step > save_at:
            _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _assert_same(run_a, _state(ag, mem, losses))
    ck_agent().save_checkpoint(str(tmp_path / "plain"))
    hp = json.load(open(tmp_path / "plain" / "rank0" / "manifest.json"))["hyper_parameters"]
    assert not {"value_transform", "value_transform_eps"} & set(hp), "default runs write the manifest of before"


@pytest.mark.parametrize("saved,live", [(dict(), VT), (VT, dict()), (VT, dict(VT, value_transform_eps=1e-2))])
def test_other_transform_is_refused(saved, live, tmp_path):
    from test_gpu_checkpoint import _refused
    small = dict(architecture="data-efficient", hidden_size=64, cuda_graph=False)
    src, mem = _agent(**saved, **small), _memory()
    for _ in range(2):
        src.reset_noise()
        src.learn(mem)
    src.save_checkpoint(str(tmp_path / "ck"), mem)
    ag, mem2 = _agent(seed=9, **live, **small), _memory()
    for _ in range(2):
        ag.reset_noise()
        ag.learn(mem2)
    _refused(ag, mem2, str(tmp_path / "ck"), match="value transform differs")
    _agent(seed=9, **saved, **small).load_checkpoint(str(tmp_path / "ck"), _memory())


@pytest.mark.parametrize("dist", list(DISTS))
def test_every_compatible_switch_graph_equals_eager(dist):
    kw = dict(VT, augment_shift=4, augment_intensity=0.05, target_tau=0.005, reset_interval=4, reset_shrink_encoder=0.5,
              weight_decay=0.1, reset_optimizer=True, redo_interval=3, learn_stats=16, **DISTS[dist])
    if dist == "categorical":
        kw.update(augment_m=2, augment_k=2)
    ga, ea = _agent(**kw), _agent(cuda_graph=False, **kw)
    gm, em = _memory(), _memory()
    for step in range(9):
        for ag, mem in ((ga, gm), (ea, em)):
            ag.reset_noise()
            ag.learn(mem)
        assert_bits_equal(cpu(ga.last_loss), cpu(ea.last_loss), f"loss of update {step}")
        _assert_snapshots(_snapshot(ga, gm), _snapshot(ea, em), f"after update {step}")
    rg, re_ = ga.learn_stats(), ea.learn_stats()
    for k in ("loss_mean", "objective", "q_mean", "target_mean"):
        assert_bits_equal(rg[k], re_[k], f"learn stats {k}")
