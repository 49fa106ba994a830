"""The learner under args.distribution = "quantile" (QR-DQN) on the GPU.

* One eager learn() per case of test_gpu_adamw.LEARNER_CASES (fused head with the online noise draw pending / flushed,
  batch 64, C3, library head): flat_grad equals float64 autograd of the QR objective through float64 copies of the online
  and target nets on the update's own batch and noise factors (bounds of DESIGN.md §4: 1e-6 head, 2e-6 conv; loss 1e-5),
  and the sum-tree leaves of the sampled indices are fl32(sqrt(loss)) of the kernel's losses, bitwise.
* Five graph replays equal five eager updates bitwise; the update graph is the categorical one with k_qr_dueling in place
  of k_c51_dueling, and the categorical graph is the default's.
* An annealed horizon (§12): each update equals the fixed-horizon update at its (n, gamma), bitwise.
* Learner statistics match float64 of the update's own rows (edge_mass NaN); act / evaluate_q / evaluate_q_memory return
  the float64 mean-quantile greedy action and value.
* Checkpoints: resume equals never stopping, bitwise; a categorical checkpoint is refused by a quantile agent and the
  reverse, changing nothing.
* Every compatible switch on at once (shift, intensity, tau, resets, AdamW with restart, ReDo, statistics): graph replays
  equal eager updates.
Deterministic cuDNN, like the other trajectory tests."""
import json

import numpy as np
import pytest
import torch

from conv_ref import conv_masks
from helpers import assert_bits_equal
from test_gpu_adamw import LEARNER_CASES
from test_gpu_augment import update_graph
from test_gpu_drq import TOL
from test_gpu_parity import DEV, FakeEnv, cpu, make_args, synthetic_ring
from update_ref import f64_forward, f64_forward_masked, qr_objective

pytestmark = pytest.mark.gpu

CAP = 8192
QR = dict(distribution="quantile", quantile_kappa=1.0)
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
                                               exp_avg_sq=o.exp_avg_sq, step_count=o.step_count, target=ag.target_flat,
                                               rng_counter=mem._rng_counter).items()}


def _assert_snapshots(a, b, what):
    for k in a:
        assert_bits_equal(a[k], b[k], f"{k} {what}")


# ---- one update against float64 autograd -----------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(LEARNER_CASES))
def test_learner_gradient_is_f64_autograd(case):
    kw, pending = LEARNER_CASES[case]
    ag, mem = _agent(cuda_graph=False, **QR, **kw), _memory()
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
        loss, obj = qr_objective(q_on[:B], q_on[B:].detach(), q_t, ws.actions, ws.returns, ws.nonterminals, ws.weights,
                                  ag.discount ** ag.n, ag.quantile_kappa)
        obj.backward()
        assert float((ag.last_loss.double() - loss.detach()).abs().max()) <= TOL["loss"], f"loss, update {step}"
        tidx, got = cpu(ws.tree_idx), cpu(ag.last_loss)
        last = np.array([i for i in range(len(tidx)) if tidx[i] not in tidx[i + 1:]])   # duplicates: the last write wins
        assert_bits_equal(cpu(mem.transitions.tree)[tidx[last]], np.sqrt(got)[last], f"priorities, update {step}")
        for n, p in on.named_parameters():
            conv = n.startswith("convs")
            off = (p.data_ptr() - opt.flat_param.data_ptr()) // 4
            d = float((opt.flat_grad[off:off + p.numel()].double() - P[n].grad.reshape(-1)).abs().max())
            assert d <= TOL["grad_conv" if conv else "grad_head"], f"gradient of {n}, update {step}: {d:.3g}"


# ---- graphs ------------------------------------------------------------------------------------------------------------------
def test_graph_replays_equal_eager_updates():
    ga, ea = _agent(**QR), _agent(cuda_graph=False, **QR)
    gm, em = _memory(), _memory()
    for step in range(7):                  # 2 eager warm-ups, the capture, 5 replays (4 + the capture's first replay)
        for ag, mem in ((ga, gm), (ea, em)):
            ag.reset_noise()
            ag.learn(mem)
        assert_bits_equal(cpu(ga.last_loss), cpu(ea.last_loss), f"loss of update {step}")
        _assert_snapshots(_snapshot(ga, gm), _snapshot(ea, em), f"after update {step}")
    assert ga._graphs and not ea._graphs


@pytest.mark.parametrize("batch", [32, 64])
def test_update_graph_swaps_only_the_loss_kernel(batch, tmp_path, monkeypatch):
    names = {}
    for tag, kw in (("default", dict()), ("categorical", dict(distribution="categorical")), ("quantile", QR)):
        names[tag] = update_graph(_agent(batch_size=batch, **kw), _memory(), tmp_path / f"{tag}.dot", monkeypatch)
    assert names["categorical"] == names["default"], "distribution 'categorical' leaves the update graph as it is"
    qr = names["quantile"]
    assert qr.count("k_qr_dueling") == names["default"].count("k_c51_dueling") == 1 and "k_c51_dueling" not in qr
    assert [("k_c51_dueling" if k == "k_qr_dueling" else k) for k in qr] == names["default"]


# ---- annealed horizon ----------------------------------------------------------------------------------------------------
def test_annealed_update_is_the_fixed_update_at_its_horizon():
    """Update u of an annealed quantile agent equals a fixed-horizon quantile agent at (n_u, gamma_u) fed the same batch
    (rb_gather at n_u on the same indices): loss and every parameter, bitwise."""
    from test_gpu_horizon import Out, lib, p, stream
    ag, plain = _agent(cuda_graph=False, **QR, **BBF), _agent(cuda_graph=False, **QR)
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


# ---- statistics, acting -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fused", [True, False], ids=["fused", "library-head"])
def test_learn_stats_match_f64(fused):
    ag, mem = _agent(learn_stats=8, fused_head=fused, cuda_graph=fused, **QR), _memory()
    for _ in range(3):
        ag.reset_noise()
        ag.learn(mem)
    torch.cuda.synchronize()
    rec = ag.learn_stats()
    assert len(rec["loss_mean"]) == 3 and np.isnan(rec["edge_mass"]).all()
    last = ag._stats["last"]
    l, w = ag.last_loss.double(), mem._last.weights.double()
    B, A, N = ag.batch_size, ag.action_space, ag.atoms
    assert rec["loss_mean"][-1] == pytest.approx(float(l.mean()), rel=1e-6)
    assert rec["objective"][-1] == pytest.approx(float((w * l).mean()), rel=1e-6, abs=1e-9)
    assert rec["loss_max"][-1] == float(l.max()) and rec["weight_min"][-1] == float(w.min())
    assert rec["target_mean"][-1] == pytest.approx(float(last["m"].double().mean()), rel=1e-5, abs=1e-6)
    if fused:
        z = last["z"][:B].double()
        q = z[:, :N].unsqueeze(1) + z[:, N:].view(B, A, N) - z[:, N:].view(B, A, N).mean(1, keepdim=True)
    else:
        q = last["q"].double()
    theta = q[torch.arange(B, device=q.device), mem._last.actions]
    assert rec["q_mean"][-1] == pytest.approx(float(theta.mean()), rel=1e-5, abs=1e-6)


def test_acting_is_the_f64_mean_quantile_greedy():
    ag = _agent(architecture="data-efficient", hidden_size=64, **QR)
    ag.eval()                                # no noise: the fused forward and the library forward see the same weights
    val, _ = synthetic_ring(256, seed=4)
    on = ag.online_net
    with torch.no_grad():
        states = val.iter_states(0, val.capacity)
        P = {n: p.detach().double() for n, p in on.named_parameters()}
        f = {n: (torch.zeros(m.in_features, device=DEV), torch.zeros(m.out_features, device=DEV))
             for n, m in on.named_children() if n.startswith("fc_")}
        q = f64_forward(on, P, f, states.double()).mean(2)              # [M][A] mean quantiles, float64
    best_v, best_a = q.max(1)
    values = torch.tensor(ag.evaluate_q_memory(val), dtype=torch.float64, device=DEV)
    assert float((values - best_v).abs().max()) <= 1e-5 * float(best_v.abs().max() + 1)
    a, v = ag.q_select(states)
    gap = q.topk(2, 1).values if q.shape[1] > 1 else None
    clear = (gap[:, 0] - gap[:, 1]) > 1e-5
    assert torch.equal(a[clear], best_a[clear]), "greedy action of the float64 means"
    for i in range(4):
        if bool(clear[i]):
            assert ag.act(states[i]) == int(best_a[i])
        assert abs(ag.evaluate_q(states[i]) - float(best_v[i])) <= 1e-5 * (abs(float(best_v[i])) + 1)


# ---- checkpoints ---------------------------------------------------------------------------------------------------------
def test_resume_equals_never_stopping(tmp_path):
    from test_gpu_checkpoint import _agent as ck_agent
    from test_gpu_checkpoint import _assert_same, _before_update, _fresh_memory, _state, _update
    from test_gpu_checkpoint import _memory as ck_memory
    kw = dict(QR, quantile_kappa=0.5)
    total, save_at = 12, 5
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
    assert (hp["distribution"], hp["quantile_kappa"]) == ("quantile", 0.5)
    ag, mem = ck_agent(seed=77, **kw), _fresh_memory()
    ag.load_checkpoint(str(tmp_path / "ck"), mem)
    for step in range(save_at, total):
        if step > save_at:
            _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _assert_same(run_a, _state(ag, mem, losses))

    ck_agent(distribution="categorical").save_checkpoint(str(tmp_path / "plain"))
    hp = json.load(open(tmp_path / "plain" / "rank0" / "manifest.json"))["hyper_parameters"]
    assert not {"distribution", "quantile_kappa"} & set(hp), "categorical runs write the manifest of before"


@pytest.mark.parametrize("saved,live", [("categorical", "quantile"), ("quantile", "categorical")])
def test_other_distribution_is_refused(saved, live, tmp_path):
    from test_gpu_checkpoint import _refused
    small = dict(architecture="data-efficient", hidden_size=64, cuda_graph=False)
    src, mem = _agent(distribution=saved, **small), _memory()
    for _ in range(2):
        src.reset_noise()
        src.learn(mem)
    src.save_checkpoint(str(tmp_path / "ck"), mem)
    ag, mem2 = _agent(seed=9, distribution=live, **small), _memory()
    for _ in range(2):
        ag.reset_noise()
        ag.learn(mem2)
    _refused(ag, mem2, str(tmp_path / "ck"), match="distribution differs")
    _agent(seed=9, distribution=saved, **small).load_checkpoint(str(tmp_path / "ck"), _memory())   # the same loads


# ---- everything on -------------------------------------------------------------------------------------------------------
def test_every_compatible_switch_graph_equals_eager():
    kw = dict(QR, augment_shift=4, augment_intensity=0.05, target_tau=0.005, reset_interval=4, reset_shrink_encoder=0.5,
              weight_decay=0.1, reset_optimizer=True, redo_interval=3, learn_stats=16)
    ga, ea = _agent(**kw), _agent(cuda_graph=False, **kw)
    gm, em = _memory(), _memory()
    for step in range(9):
        for ag, mem in ((ga, gm), (ea, em)):
            ag.reset_noise()
            ag.learn(mem)
        assert_bits_equal(cpu(ga.last_loss), cpu(ea.last_loss), f"loss of update {step}")
        _assert_snapshots(_snapshot(ga, gm), _snapshot(ea, em), f"after update {step}")
    assert ga._graphs and not ea._graphs and ga.reset_count == ea.reset_count == 2 and ga.redo_count == 3
    rg, re_ = ga.learn_stats(), ea.learn_stats()
    for k in ("loss_mean", "objective", "q_mean", "target_mean", "grad_norm"):
        assert_bits_equal(rg[k], re_[k], f"learn stats {k}")
