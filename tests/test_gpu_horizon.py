"""BBF's annealed update horizon (rainbow_b200.horizon, rb_horizon_advance, rb_gather_horizon, args.anneal_steps) on the GPU.

* rb_horizon_advance copies row min(u, T) bitwise and advances the counter, eagerly and as a graph replay.
* rb_gather_horizon with the row (n_t, gamma) equals rb_gather / rb_gather_shift / rb_gather_aug at n = n_t with gamma_pow
  = fl32(gamma ** k) on the same indices, bitwise, for every n_t in 1 .. n_max and three gammas, on a replay with short
  episodes and windows across the ring's wrap; its nonterminals are fl32(nonterminal * gamma ** n_t).  And the oracle's
  gather agrees.
* The discount-form nonterminals with gamma_n = 1 give every loss kernel's loss, gradient and m bitwise.
* The learner: a constant schedule is an agent without the options; an annealed agent's update u equals a plain agent
  at (n_u, gamma_u) fed the same batch; graph replays equal eager updates; resets restart the schedule; a resumed run
  equals an uninterrupted one; the update graph gains one rb_horizon_advance node and swaps the gather.
Deterministic cuDNN, like the other trajectory tests."""
import json

import numpy as np
import pytest
import torch

from helpers import assert_bits_equal
from test_gpu_augment import episodic_memory, update_graph
from test_gpu_parity import DEV, FakeEnv, cpu, make_args, synthetic_ring

pytestmark = pytest.mark.gpu
CAP = 8192
BBF = dict(anneal_steps=6, multi_step_start=10, discount_start=0.97, multi_step=3, discount=0.997)


@pytest.fixture(autouse=True)
def deterministic_cudnn():
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = old


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


def stream():
    return torch.cuda.current_stream().cuda_stream


def p(t):
    return None if t is None else t.data_ptr()


def row_tensor(n, g):
    """One rb_horizon row for a fixed (n, gamma), on the device."""
    from rainbow_b200.horizon import ROW_DTYPE
    r = np.zeros(1, dtype=ROW_DTYPE)
    r["n"], r["gamma_n"] = n, np.float32(g ** n)
    r["gamma_pow"][0, :n] = np.array([g ** k for k in range(n)]).astype(np.float32)
    return torch.from_numpy(r.view(np.uint8).copy()).to(DEV)


# ---- rb_horizon_advance ----------------------------------------------------------------------------------------------------
def test_advance_copies_the_clamped_row_and_counts():
    from rainbow_b200.horizon import HorizonSchedule
    T = 6
    hz = HorizonSchedule(T, 10, 3, 0.97, 0.997, DEV)
    for u in (0, 1, T - 1, T, T + 3):
        hz.set_step(u)
        hz.advance()
        torch.cuda.synchronize()
        assert cpu(hz.current).tobytes() == hz.rows[min(u, T)].tobytes(), f"row of step {u}"
        assert int(hz.counter.item()) == u + 1 and hz.step == u + 1
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g):
            hz.advance()
    torch.cuda.current_stream().wait_stream(s)
    for u in (0, 1, T - 1, T, T + 3):
        hz.set_step(u)
        hz.current.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert cpu(hz.current).tobytes() == hz.rows[min(u, T)].tobytes(), f"graph replay, row of step {u}"
        assert int(hz.counter.item()) == u + 1


# ---- rb_gather_horizon -----------------------------------------------------------------------------------------------------
class Out:
    def __init__(self, B, history, M=1, K=1, copies=1):
        self.B = B
        self.states = torch.full((M * B, history, 84, 84), float("nan"), device=DEV)
        self.next_states = torch.full((K * B, history, 84, 84), float("nan"), device=DEV)
        self.actions = torch.full((B,), -1, dtype=torch.int64, device=DEV)
        self.returns = torch.full((B,), float("nan"), device=DEV)
        self.nonterminals = torch.full((B,), float("nan"), device=DEV)
        self.shifts = torch.full((2 * copies * B * 2,), -7, dtype=torch.int32, device=DEV)
        self.scales = torch.full((2 * copies * B,), float("nan"), device=DEV)

    def host(self):
        return {k: cpu(getattr(self, k)) for k in ("states", "next_states", "actions", "returns", "nonterminals", "shifts",
                                                    "scales")}


def _common(mem, didx, out, n, gp):
    tr = mem.transitions
    return (p(tr.frames), p(tr.timestep), p(tr.action), p(tr.reward), p(tr.nonterminal), tr.size, p(didx), out.B,
            mem.history, n, p(gp), p(out.states), p(out.next_states), p(out.actions), p(out.returns), p(out.nonterminals))


AUG = {"plain": (0, 0.0, 1, 1), "shift4": (4, 0.0, 1, 1), "aug-p4-i0.05-m2-k2": (4, 0.05, 2, 2)}


@pytest.mark.parametrize("aug", list(AUG))
def test_gather_horizon_is_the_fixed_gather_at_every_n(aug):
    import oracle
    pad, intensity, M, K = AUG[aug]
    n_max, history, B = 10, 4, 48
    mem, ts = episodic_memory(history, n_max, cap=4096, seed=2)
    cap = mem.capacity
    rs = np.random.RandomState(11)
    idx = rs.randint(0, cap, B)
    idx[:4] = [0, 1, cap - 1, cap - 5]                                  # windows across the ring's wrap
    idx[4:12] = rs.choice(np.flatnonzero(ts == 1), 8)                   # episode starts inside the window
    idx[12:20] = rs.choice(np.flatnonzero(ts == 0), 8)
    didx = torch.from_numpy(idx.astype(np.int64)).to(DEV)
    counter = torch.tensor([(5 << 32) + 77], dtype=torch.int64, device=DEV)
    seed = 0x1234567
    copies = max(M, K)
    ref_tree = None
    if aug == "plain":
        tr = mem.transitions
        ref_tree = oracle.OracleTree(cap)
        for name in ("frames", "timestep", "action", "reward", "nonterminal"):
            getattr(ref_tree, name)[:] = cpu(getattr(tr, name)).reshape(getattr(ref_tree, name).shape)
    blanked_nt = False
    for g in (0.97, 0.99, 0.997):
        for n in range(1, n_max + 1):
            gp = torch.tensor([g ** k for k in range(n)], dtype=torch.float32, device=DEV)
            row = row_tensor(n, g)
            want, got = Out(B, history, M, K, copies), Out(B, history, M, K, copies)
            c = _common(mem, didx, want, n, gp)
            if aug == "plain":
                rc = lib().rb_gather(*c, stream())
            elif aug == "shift4":
                rc = lib().rb_gather_shift(*c, pad, seed, p(counter), p(want.shifts), stream())
            else:
                rc = lib().rb_gather_aug(*c, pad, intensity, M, K, seed, p(counter), p(want.shifts), p(want.scales),
                                         stream())
            assert rc == 0, lib().rb_last_error()
            h = _common(mem, didx, got, n_max, row)
            rc = lib().rb_gather_horizon(*h, pad, intensity, M, K, seed, p(counter), p(got.shifts), p(got.scales), stream())
            assert rc == 0, lib().rb_last_error()
            torch.cuda.synchronize()
            a, b = want.host(), got.host()
            for k in ("states", "next_states", "actions", "returns", "shifts", "scales"):
                assert_bits_equal(b[k], a[k], f"{k}, n {n}, gamma {g}")
            assert_bits_equal(b["nonterminals"], (a["nonterminals"] * np.float32(g ** n)).astype(np.float32),
                              f"nonterminals in discount form, n {n}, gamma {g}")
            blanked_nt = blanked_nt or bool((a["nonterminals"] == 0).any())
            if ref_tree is not None and g == 0.99:
                s, act, ret, ns, nt = oracle.gather(ref_tree, idx, history, n, cpu(gp))
                assert_bits_equal(b["states"], s, "oracle states")
                assert_bits_equal(b["next_states"], ns, "oracle next states")
                assert_bits_equal(b["returns"], ret, "oracle returns")
                assert_bits_equal(b["nonterminals"], (nt.reshape(-1) * np.float32(g ** n)).astype(np.float32), "oracle nt")
    assert blanked_nt, "the fixture has windows whose last record is blanked or terminal"


def test_gather_horizon_refusals_launch_nothing():
    mem, _ = episodic_memory(4, 10, cap=1024)
    B = 8
    didx = torch.zeros(B, dtype=torch.int64, device=DEV)
    out = Out(B, 4, 2, 2, 2)
    row = row_tensor(3, 0.99)
    ctr = torch.zeros(1, dtype=torch.int64, device=DEV)
    L = lib()

    def call(n_max=10, cur=row, pad=0, intensity=0.0, M=1, K=1, counter=ctr, shifts=out.shifts, scales=out.scales):
        return L.rb_gather_horizon(*_common(mem, didx, out, n_max, cur), pad, intensity, M, K, 1, p(counter), p(shifts),
                                   p(scales), stream())
    assert call(cur=None) == -22
    assert call(n_max=61) == -34 and call(n_max=0) == -22
    assert call(pad=-1) == -34 and call(pad=17) == -34
    assert call(intensity=float("nan")) == -34 and call(intensity=0.6) == -34
    assert call(M=0) == -34 and call(K=9) == -34
    assert call(pad=4, counter=None) == -22 and call(pad=4, shifts=None) == -22
    assert call(pad=4, M=2, scales=None) == -22
    assert call(pad=4, scales=None) == 0 and call() == 0
    table = torch.zeros(264 * 3, dtype=torch.uint8, device=DEV)
    assert L.rb_horizon_advance(None, 2, p(ctr), p(row), stream()) == -22
    assert L.rb_horizon_advance(p(table), 2, None, p(row), stream()) == -22
    assert L.rb_horizon_advance(p(table), 2, p(ctr), None, stream()) == -22
    assert L.rb_horizon_advance(p(table), 0, p(ctr), p(row), stream()) == -34
    assert L.rb_horizon_advance(p(table), 65537, p(ctr), p(row), stream()) == -34
    torch.cuda.synchronize()
    assert int(ctr.item()) == 0


# ---- the loss kernels on discount-form nonterminals ------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["c51-z51", "c51-z101", "dueling", "dueling-avg"])
def test_discount_form_gives_the_fixed_gamma_loss(variant):
    from rainbow_b200 import agent as A
    torch.manual_seed(3)
    B, acts, g, n = 32, 6, 0.97, 7
    Z = 101 if variant == "c51-z101" else 51
    support = torch.linspace(-10.0, 10.0, Z, device=DEV)
    dz_ = 20.0 / (Z - 1)
    nt01 = (torch.rand(B, 1, device=DEV) > 0.3).float()
    disc = nt01 * np.float32(g ** n)
    gamma_n = g ** n
    actions = torch.randint(0, acts, (B,), device=DEV)
    returns = torch.randn(B, device=DEV) * 3
    weights = torch.rand(B, device=DEV)
    outs = []
    for nt, gn in ((nt01, gamma_n), (disc, 1.0)):
        m = torch.empty((B, Z), device=DEV)
        if variant.startswith("c51"):
            gen = torch.Generator(device=DEV).manual_seed(9)
            q = [torch.randn((B, acts, Z), device=DEV, generator=gen) for _ in range(3)]
            loss, grad = A.c51_loss_grad(*q, actions, returns, nt, weights, support, -10.0, 10.0, dz_, gn, m_out=m)
        else:
            M, K = (2, 2) if variant == "dueling-avg" else (1, 1)
            gen = torch.Generator(device=DEV).manual_seed(9)
            zo = torch.randn(((M + K) * B, Z * (1 + acts)), device=DEV, generator=gen)
            zt = torch.randn((K * B, Z * (1 + acts)), device=DEV, generator=gen)
            if variant == "dueling":
                loss, grad = A.c51_dueling_loss_grad(zo, zt, acts, Z, actions, returns, nt, weights, support, -10.0, 10.0,
                                                     dz_, gn, m_out=m)
            else:
                loss, grad = A.c51_dueling_avg_loss_grad(zo, zt, acts, Z, actions, returns, nt, weights, support, -10.0,
                                                         10.0, dz_, gn, M, K, m_out=m)
        torch.cuda.synchronize()
        outs.append((cpu(loss), cpu(grad), cpu(m)))
    for k, name in enumerate(("loss", "gradient", "m")):
        assert_bits_equal(outs[1][k], outs[0][k], name)
    assert (cpu(nt01) == 0).any() and (cpu(nt01) == 1).any()


# ---- the learner -----------------------------------------------------------------------------------------------------------
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


def test_option_checks():
    for bad in (dict(anneal_steps=65537), dict(anneal_steps=-1), dict(anneal_steps=2.5), dict(anneal_steps=3, multi_step_start=0),
                dict(anneal_steps=3, discount_start=1.0), dict(multi_step_start=5), dict(discount_start=0.9),
                dict(anneal_steps=3, multi_step_start=61)):
        with pytest.raises(ValueError):
            _agent(**bad)


@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
def test_constant_schedule_is_the_plain_agent(use_graph):
    const = dict(anneal_steps=4, multi_step_start=3, discount_start=0.99)
    a, b = _agent(cuda_graph=use_graph, **const), _agent(cuda_graph=use_graph)
    ma, mb = _memory(**const), _memory()
    for step in range(7 if use_graph else 5):
        for ag, mem in ((a, ma), (b, mb)):
            ag.reset_noise()
            ag.learn(mem)
        assert_bits_equal(cpu(a.last_loss), cpu(b.last_loss), f"loss of update {step}")
        assert a.horizon() == (3, 0.99)
    assert bool(a._graphs) == use_graph
    _assert_snapshots(_snapshot(a, ma), _snapshot(b, mb), "constant schedule vs no schedule")


C3 = dict(architecture="data-efficient", hidden_size=256)
LEARNER_CASES = {
    "fused-pending": (dict(), True),
    "fused-flushed": (dict(), False),
    "batch64": (dict(batch_size=64), True),
    "c3": (C3, True),
    "library-head": (dict(fused_head=False), False),
}


@pytest.mark.parametrize("case", list(LEARNER_CASES))
def test_annealed_update_is_the_plain_update_at_its_horizon(case):
    """Update u of an annealed agent (T 6, n 10 -> 3, gamma 0.97 -> 0.997) equals a plain agent at (n_u, gamma_u) fed the
    same sampled batch (rb_gather at n_u on the same indices) through _update_from_batch: loss and every parameter."""
    from rainbow_b200.horizon import horizon_at
    kw, pending = LEARNER_CASES[case]
    ag, plain = _agent(cuda_graph=False, **BBF, **kw), _agent(cuda_graph=False, **kw)
    assert ag._fused_path(ag.batch_size) == (case != "library-head")
    mem = _memory(**BBF)
    assert mem.n == 10
    seen = set()
    for u in range(8):
        n_u, g_u = ag.horizon()
        assert (n_u, g_u) == horizon_at(u, 6, 10, 3, 0.97, 0.997)
        seen.add(n_u)
        for a in (ag, plain):
            a.reset_noise()
            if not pending:
                a.online_net.flush_noise()
        ag.learn(mem)
        ws = mem._last
        B = ws.B
        gp = torch.tensor([g_u ** k for k in range(n_u)], dtype=torch.float32, device=DEV)
        out = Out(B, 4)
        tr = mem.transitions
        rc = lib().rb_gather(p(tr.frames), p(tr.timestep), p(tr.action), p(tr.reward), p(tr.nonterminal), tr.size,
                             p(ws.data_idx), B, 4, n_u, p(gp), p(out.states), p(out.next_states), p(out.actions),
                             p(out.returns), p(out.nonterminals), stream())
        assert rc == 0
        both = torch.cat([out.states, out.next_states])
        batch = (ws.tree_idx.clone(), both[:B], out.actions, out.returns, both[B:], out.nonterminals.view(B, 1),
                 ws.weights.clone())
        plain.n, plain.discount = n_u, g_u
        loss = plain._update_from_batch(batch, gate=ws.status)
        torch.cuda.synchronize()
        assert_bits_equal(cpu(ag.last_loss), cpu(loss), f"loss of update {u}")
        for name in ("flat_param", "exp_avg", "exp_avg_sq"):
            assert_bits_equal(cpu(getattr(ag.optimiser, name)), cpu(getattr(plain.optimiser, name)), f"{name} after {u}")
    assert seen == {10, 8, 7, 5, 4, 3}


def test_annealed_graph_replays_equal_eager_updates():
    ga, ea = _agent(**BBF), _agent(cuda_graph=False, **BBF)
    gm, em = _memory(**BBF), _memory(**BBF)
    for step in range(9):
        for ag, mem in ((ga, gm), (ea, em)):
            ag.reset_noise()
            ag.learn(mem)
        assert_bits_equal(cpu(ga.last_loss), cpu(ea.last_loss), f"loss of update {step}")
        assert ga.horizon() == ea.horizon()
    assert ga._graphs and not ea._graphs
    assert int(ga._horizon.counter.item()) == ga._horizon.step == 9
    _assert_snapshots(_snapshot(ga, gm), _snapshot(ea, em), "graph vs eager")


@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
def test_resets_restart_the_schedule(use_graph):
    from rainbow_b200.horizon import horizon_at
    ag, mem = _agent(cuda_graph=use_graph, reset_interval=4, **BBF), _memory(**BBF)
    for k in range(10):
        assert ag.horizon() == horizon_at(k % 4, 6, 10, 3, 0.97, 0.997), f"before learn() {k}"
        ag.reset_noise()
        ag.learn(mem)
        torch.cuda.synchronize()
        assert int(ag._horizon.counter.item()) == ag._horizon.step == (k + 1) % 4
    assert ag.reset_count == 2
    ag.reset_parameters()
    assert ag.horizon() == (10, 0.97) and int(ag._horizon.counter.item()) == 0


def test_resume_equals_never_stopping(tmp_path):
    """anneal on, tau 0.005, a reset every 6 updates: 5 updates, save, fresh objects, load, 7 more == 12 uninterrupted."""
    from rainbow_b200.memory import ReplayMemory
    kw = dict(target_tau=0.005, reset_interval=6, **BBF)

    def run(ag, mem, steps, losses):
        for _ in steps:
            ag.reset_noise()
            ag.learn(mem)
            losses.append(ag.last_loss.clone())

    ag, mem = _agent(**kw), _memory(**BBF)
    la = []
    run(ag, mem, range(12), la)
    a = dict(_snapshot(ag, mem), losses=cpu(torch.stack(la)))
    ag, mem = _agent(**kw), _memory(**BBF)
    lb = []
    run(ag, mem, range(5), lb)
    ag.save_checkpoint(str(tmp_path / "ck"), mem)
    man = json.load(open(tmp_path / "ck" / "rank0" / "manifest.json"))
    hp = man["hyper_parameters"]
    assert (hp["anneal_steps"], hp["multi_step_start"], hp["discount_start"]) == (6, 10, 0.97)
    assert man["learner"]["horizon_step"] == 5
    ag, mem = _agent(seed=77, **kw), ReplayMemory(make_args(**BBF), CAP, seed=12345)
    ag.load_checkpoint(str(tmp_path / "ck"), mem)
    assert ag._horizon.step == 5 and int(ag._horizon.counter.item()) == 5
    run(ag, mem, range(5, 12), lb)
    b = dict(_snapshot(ag, mem), losses=cpu(torch.stack(lb)))
    _assert_snapshots(a, b, "resumed vs uninterrupted")


@pytest.mark.parametrize("batch", [32, 64])
def test_update_graph_adds_the_advance_and_swaps_the_gather(batch, tmp_path, monkeypatch):
    plain = update_graph(_agent(batch_size=batch), _memory(), tmp_path / "plain.dot", monkeypatch)
    on = update_graph(_agent(batch_size=batch, **BBF), _memory(**BBF), tmp_path / "on.dot", monkeypatch)
    assert on.count("k_horizon_advance") == 1 and "k_horizon_advance" not in plain
    assert on.count("k_gather_hz") == plain.count("k_gather") == 1 and "k_gather" not in on
    rest = [("k_gather" if k == "k_gather_hz" else k) for k in on if k != "k_horizon_advance"]
    assert rest == plain
