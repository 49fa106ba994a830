"""Bootstrapping through time-limit truncations on the device, bitwise:

* rb_gather_trunc without augmentation against tests/trunc_ref.py over history 1 and 4, n = 1, 3, 20, 36 and every cut
  k in 1 .. n - 1 (a final observation at the ring's wrap and two short episodes in one window among them), eager and as
  a graph replay, guard rows untouched; with an annealed row (n_t < n_max) against the reference at n = n_t;
* its shift and aug forms (M = 2, K = 3) against rb_gather_horizon at a row of n = k for the cut samples, with the same
  draws, and at n for the rest;
* append_truncated, immediate and deferred, against the oracle's ring: frames, timestep, action, reward, nonterminal,
  leaves (0 at F), running max, host mirrors;
* the device sampler never returns a final observation;
* the loss kernels on a cut sample's discount-form nonterminal equal the fixed-horizon loss at gamma_k;
* the learner: graph replays equal eager updates with final observations in the ring, the update graph keeps its nodes
  with only the gather swapped, and a resume from a checkpoint taken with final observations in the ring equals never
  stopping; a replay without the switch refuses that checkpoint."""

import numpy as np
import pytest
import torch

import oracle
import trunc_ref
from helpers import assert_bits_equal
from test_gpu_horizon import _assert_snapshots, _snapshot
from test_gpu_augment import update_graph
from test_gpu_parity import DEV, FakeEnv, cpu, make_args, synthetic_ring
from test_gpu_replay_data import DeviceRing, GatherOut, assert_gather_equals_oracle, eager_and_graph, gather_args
from test_truncation_host import GRID, GAMMA, cut_cases

pytestmark = pytest.mark.gpu
RB_ERR_INVAL, RB_ERR_RANGE = -22, -34


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


def row(n, g, n_row=None):
    """The rb_horizon row of a horizon of n steps at discount g (n field n_row when given)."""
    from rainbow_b200.horizon import ROW_DTYPE
    r = np.zeros(1, dtype=ROW_DTYPE)
    r["n"], r["gamma_n"] = n if n_row is None else n_row, np.float32(g ** n)
    r["gamma_pow"][0, :n] = np.array([g ** k for k in range(n)]).astype(np.float32)
    return torch.from_numpy(r.view(np.uint8).copy()).to(DEV), r["gamma_pow"][0].copy(), np.float32(g ** n)


# ---- rb_gather_trunc, no augmentation ----------------------------------------------------------------------------------
@pytest.mark.parametrize("H,n", GRID, ids=lambda v: str(v))
def test_gather_trunc_equals_the_reference(H, n):
    t, idx, want_k = cut_cases(H, n, 10 * H + n)
    ring = DeviceRing(t)
    didx = torch.from_numpy(idx).to(DEV)
    r, gp, gn = row(n, GAMMA)
    B = idx.size
    out = eager_and_graph(lambda o: lib().rb_gather_trunc(*gather_args(ring, didx, H, n, r, o), 0, 0.0, 1, 1, 0, None,
                                                          None, None, stream()), B, H)
    s, a, ret, ns, nt, k = trunc_ref.gather_trunc(t, idx, H, n, gp[:n], gn)
    assert_bits_equal(k, want_k, "cuts")
    got_nt, _ = assert_gather_equals_oracle(out, (s, a, ret, ns, nt), f"H {H} n {n}")
    assert_bits_equal(got_nt, nt.reshape(-1), "nonterminals")


@pytest.mark.parametrize("H,n_max,n_t", [(4, 20, 3), (4, 36, 10), (1, 20, 7)], ids=lambda v: str(v))
def test_gather_trunc_at_an_annealed_row(H, n_max, n_t):
    """A row of n_t < n_max: the cut is looked for in (t, t + n_t) and the rest is the reference at n = n_t."""
    t, idx, _ = cut_cases(H, n_max, 10 * H + n_max)
    ring = DeviceRing(t)
    didx = torch.from_numpy(idx).to(DEV)
    r, gp, gn = row(n_t, 0.995)
    out = eager_and_graph(lambda o: lib().rb_gather_trunc(*gather_args(ring, didx, H, n_max, r, o), 0, 0.0, 1, 1, 0, None,
                                                          None, None, stream()), idx.size, H)
    s, a, ret, ns, nt, k = trunc_ref.gather_trunc(t, idx, H, n_t, gp[:n_t], gn)
    assert (k < n_t).any() and (k == n_t).any()
    got_nt, _ = assert_gather_equals_oracle(out, (s, a, ret, ns, nt), f"n_t {n_t}")
    assert_bits_equal(got_nt, nt.reshape(-1), "nonterminals")


def test_gather_trunc_refusals_write_nothing():
    t, idx, _ = cut_cases(4, 3, 43)
    ring = DeviceRing(t)
    didx = torch.from_numpy(idx).to(DEV)
    r, _, _ = row(3, GAMMA)
    for H, n, cur, pad, code in ((32, 33, r, 0, RB_ERR_RANGE), (4, 3, None, 0, RB_ERR_INVAL), (4, 3, r, 17, RB_ERR_RANGE),
                                 (4, 3, r, 4, RB_ERR_INVAL)):
        out = GatherOut(idx.size, H)
        rc = lib().rb_gather_trunc(*gather_args(ring, didx, H, n, cur, out), pad, 0.0, 1, 1, 0, None, None, None, stream())
        assert rc == code, (H, n, pad)
        torch.cuda.synchronize()
        out.assert_untouched(f"refused H {H} n {n} pad {pad}")


# ---- shift and aug forms against rb_gather_horizon at n = k ---------------------------------------------------------------
class AugOut:
    def __init__(self, B, H, M, K):
        self.B, self.M, self.K = B, M, K
        c = max(M, K)
        self.states = torch.full((M * B + 2, H, 84, 84), float("nan"), device=DEV)
        self.next_states = torch.full((K * B + 2, H, 84, 84), float("nan"), device=DEV)
        self.actions = torch.full((B + 2,), -7, dtype=torch.int64, device=DEV)
        self.returns = torch.full((B + 2,), float("nan"), device=DEV)
        self.nonterminals = torch.full((B + 2,), float("nan"), device=DEV)
        self.shifts = torch.full((2 * c * B * 2 + 4,), -7, dtype=torch.int32, device=DEV)
        self.scales = torch.full((2 * c * B + 4,), float("nan"), device=DEV)

    def launch(self, fn, ring, didx, H, n_max, r, pad, intensity, ctr):
        return fn(p(ring.frames), p(ring.timestep), p(ring.action), p(ring.reward), p(ring.nonterminal), ring.size, p(didx),
                  self.B, H, n_max, p(r), p(self.states), p(self.next_states), p(self.actions), p(self.returns),
                  p(self.nonterminals), pad, intensity, self.M, self.K, 1234, p(ctr), p(self.shifts), p(self.scales),
                  stream())

    def rows(self, x, copies, sel):
        return cpu(x[:copies * self.B].reshape(copies, self.B, *x.shape[1:])[:, sel])

    def guards(self):
        for x, end in ((self.states, self.M * self.B), (self.next_states, self.K * self.B), (self.actions, self.B),
                       (self.returns, self.B), (self.nonterminals, self.B)):
            g = x[end:]
            assert bool((g == -7).all() if g.dtype == torch.int64 else torch.isnan(g).all()), "a guard row was written"


@pytest.mark.parametrize("H,n", [(4, 3), (4, 20), (1, 36)], ids=lambda v: str(v))
@pytest.mark.parametrize("aug", ["shift", "aug"])
def test_gather_trunc_augmented_equals_the_horizon_gather_at_k(H, n, aug):
    t, idx, _ = cut_cases(H, n, 10 * H + n)
    ring = DeviceRing(t)
    didx = torch.from_numpy(idx).to(DEV)
    B = idx.size
    pad, intensity, M, K = (4, 0.0, 1, 1) if aug == "shift" else (4, 0.05, 2, 3)
    ctr = torch.tensor([77], dtype=torch.int64, device=DEV)
    r, gp, gn = row(n, GAMMA)
    got = AugOut(B, H, M, K)
    assert got.launch(lib().rb_gather_trunc, ring, didx, H, n, r, pad, intensity, ctr) == 0, lib().rb_last_error()
    torch.cuda.synchronize()
    got.guards()
    k = trunc_ref.gather_trunc(t, idx, H, n, gp[:n], gn)[5]
    assert (k < n).sum() >= n - 1
    for kk in sorted(set(k.tolist())):
        sel = np.flatnonzero(k == kk)
        rk, _, gk = row(kk, GAMMA)
        want = AugOut(B, H, M, K)
        assert want.launch(lib().rb_gather_horizon, ring, didx, H, n, rk, pad, intensity, ctr) == 0
        torch.cuda.synchronize()
        what = f"{aug} H {H} n {n} k {kk}"
        assert_bits_equal(got.rows(got.states, M, sel), want.rows(want.states, M, sel), f"{what}: states")
        assert_bits_equal(got.rows(got.next_states, K, sel), want.rows(want.next_states, K, sel), f"{what}: next states")
        for name in ("actions", "returns", "nonterminals"):
            assert_bits_equal(cpu(getattr(got, name))[sel], cpu(getattr(want, name))[sel], f"{what}: {name}")
        assert_bits_equal(cpu(got.shifts), cpu(want.shifts), f"{what}: shifts")
        if aug == "aug":
            assert_bits_equal(cpu(got.scales), cpu(want.scales), f"{what}: scales")


# ---- append_truncated --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("deferred", [False, True], ids=["immediate", "deferred"])
@pytest.mark.parametrize("host_frames", [False, True], ids=["device", "host"])
def test_append_truncated_equals_the_oracle(deferred, host_frames):
    from rainbow_b200.memory import ReplayMemory
    size = 64
    mem = ReplayMemory(make_args(bootstrap_truncation=True), size, defer_appends=deferred)
    ot = oracle.OracleTree(size)
    rs = np.random.RandomState(5)
    mem.update_priorities(np.arange(size) + ot.tree_start, np.full(size, 2.0, np.float32))   # running max 2^0.5
    ot.update(np.arange(size) + ot.tree_start, oracle.pow_priorities(np.full(size, 2.0, np.float32), 0.5))
    t_ep = 0
    for step in range(150):   # wraps the ring twice
        st = rs.uniform(0, 1, (4, 84, 84)).astype(np.float32)
        state = torch.from_numpy(st) if host_frames else torch.from_numpy(st).to(DEV)
        a, rew, u = int(rs.randint(0, 6)), float(rs.uniform(-1, 1)), rs.uniform()
        if u < 0.1:
            fin = rs.uniform(0, 1, (4, 84, 84)).astype(np.float32)
            mem.append_truncated(state, a, rew, torch.from_numpy(fin) if host_frames else torch.from_numpy(fin).to(DEV))
            ot.append(t_ep, oracle.quantise_frame(st[-1]), a, np.float32(rew), True)
            f = ot.index
            ot.append(t_ep + 1, oracle.quantise_frame(fin[-1]), 0, np.float32(0), True, value=0.0)
            ot.nonterminal[f] = trunc_ref.FINAL
            t_ep = 0
        else:
            term = u > 0.93
            mem.append(state, a, rew, term)
            ot.append(t_ep, oracle.quantise_frame(st[-1]), a, np.float32(rew), not term)
            t_ep = 0 if term else t_ep + 1
        assert mem.transitions.index == ot.index and mem.t == t_ep
    mem.flush_appends()
    tr = mem.transitions
    torch.cuda.synchronize()
    assert (ot.nonterminal == trunc_ref.FINAL).sum() >= 5
    for name in ("frames", "timestep", "action", "reward", "nonterminal"):
        assert_bits_equal(cpu(getattr(tr, name)).reshape(getattr(ot, name).shape), getattr(ot, name), name)
    assert_bits_equal(tr.sum_tree, ot.sum_tree, "tree")
    assert tr.max == float(ot.max[0])
    assert (tr.sum_tree[ot.tree_start + np.flatnonzero(ot.nonterminal == trunc_ref.FINAL)] == 0).all()
    assert int(tr.ring_state[2].item()) == t_ep and int(tr.ring_state[0].item()) == ot.index
    got = tr.get(np.arange(size))
    assert_bits_equal(got["final"], ot.nonterminal == trunc_ref.FINAL, "get() final")


def test_the_sampler_never_returns_a_final_observation():
    from rainbow_b200.memory import _SampleWorkspace
    mem, _ = synthetic_ring(4096, seed=3, args=dict(bootstrap_truncation=True))
    tr = mem.transitions
    nt = cpu(tr.nonterminal).copy()
    ts = cpu(tr.timestep).copy()
    final = np.arange(5, 4096, 7)
    final = final[(final != tr.index - 1) & (final != tr.index)]
    nt[final] = trunc_ref.FINAL
    ts[(final + 1) % 4096] = 0
    tr.load_arrays(nonterminal=nt, timestep=ts, t_episode=int(ts[tr.index - 1]) + 1)
    mem.update_priorities(final + tr.tree_start, np.zeros(final.size, np.float32))
    ws = _SampleWorkspace(512, 4, mem.device)
    seen = []
    for _ in range(200):
        mem.sample_into(ws)
        seen.append(ws.data_idx.clone())
    torch.cuda.synchronize()
    got = cpu(torch.cat(seen))
    assert not np.isin(got, final).any(), "a final observation was sampled"
    assert np.isin((got[:, None] + np.arange(1, 3)) % 4096, final).any()   # cut windows were sampled


# ---- the loss kernels on a cut sample's nonterminal ----------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["c51", "c51-vt", "c51-risk", "qr", "qr-vt", "qr-risk", "qr-munchausen"])
def test_discount_form_at_k_gives_the_fixed_horizon_loss(variant):
    """Rows cut at k with nonterminal fl32(nt gamma^k) under gamma_n = 1 give the loss, priorities and gradient rows the
    kernel gives on 0 / 1 nonterminals under gamma_n = gamma^k."""
    from rainbow_b200 import agent as A
    torch.manual_seed(3)
    B, acts, n = 32, 6, 5
    Z = 51 if variant.startswith("c51") else 32
    gen = torch.Generator(device=DEV).manual_seed(9)
    q = [torch.randn((B, acts, Z), device=DEV, generator=gen) for _ in range(3)]
    k = torch.from_numpy(np.arange(B) % n + 1)
    nt01 = (torch.rand(B, 1) > 0.2).float()
    gk = torch.from_numpy(np.array([np.float32(GAMMA ** int(j)) for j in k], np.float32)).reshape(B, 1)
    disc = (nt01 * gk).to(DEV)
    actions = torch.randint(0, acts, (B,), device=DEV)
    returns = torch.randn(B, device=DEV) * 3
    weights = torch.rand(B, device=DEV)
    support = torch.linspace(-10.0, 10.0, Z, device=DEV)

    def run(nt, gamma_n):
        if variant.startswith("c51"):
            kw = dict(eps=1e-3, support_q=support) if variant == "c51-vt" else {}
            if variant == "c51-risk":
                kw = dict(risk=(1, 0.25))
            loss, grad = A.c51_loss_grad(*q, actions, returns, nt, weights, support, -10.0, 10.0, 20.0 / (Z - 1),
                                         gamma_n, **kw)
        elif variant == "qr-munchausen":
            loss, grad = A.qr_munchausen_loss_grad(*q, actions, returns, nt, weights, 1.0, gamma_n, 0.9, 0.03, -1.0)
        else:
            kw = dict(eps=1e-3) if variant == "qr-vt" else dict(risk=(1, 0.25)) if variant == "qr-risk" else {}
            loss, grad = A.qr_loss_grad(*q, actions, returns, nt, weights, 1.0, gamma_n, **kw)
        torch.cuda.synchronize()
        return cpu(loss), cpu(grad)

    got = run(disc, 1.0)
    for kk in range(1, n + 1):
        sel = np.flatnonzero(k.numpy() == kk)
        want = run(nt01.to(DEV), GAMMA ** kk)
        assert_bits_equal(got[0][sel], want[0][sel], f"{variant} k {kk}: loss")
        assert_bits_equal(got[1][sel], want[1][sel], f"{variant} k {kk}: gradient")


# ---- the learner ---------------------------------------------------------------------------------------------------------
CAP = 8192


def _agent(seed=5, **kw):
    from rainbow_b200.agent import Agent
    torch.manual_seed(seed)
    return Agent(make_args(**kw), FakeEnv(6))


def _memory(**args):
    """synthetic_ring with a final observation about every 9 records (leaf 0, an episode start after it)."""
    mem, _ = synthetic_ring(CAP, seed=3, args=args)
    mem.seed = 99
    if args.get("bootstrap_truncation"):
        tr = mem.transitions
        nt, ts = cpu(tr.nonterminal).copy(), cpu(tr.timestep).copy()
        head = tr.index
        final = np.arange(3, CAP, 9)
        final = final[np.abs(final - head) > 2]
        nt[final], nt[final - 1] = trunc_ref.FINAL, 1
        ts[(final + 1) % CAP] = 0
        tr.load_arrays(nonterminal=nt, timestep=ts, t_episode=int(ts[head - 1]) + 1)
        mem.update_priorities(final + tr.tree_start, np.zeros(final.size, np.float32))
    return mem


TRUNC = dict(bootstrap_truncation=True)


@pytest.mark.parametrize("kw", [dict(), dict(distribution="quantile", atoms=32), dict(munchausen=True,
                                distribution="quantile", atoms=32), dict(value_transform="rescale"), dict(risk_measure="cvar",
                                risk_eta=0.25), dict(anneal_steps=6, multi_step_start=10, discount_start=0.97,
                                multi_step=3, discount=0.997)], ids=["c51", "qr", "munchausen", "vt", "risk", "horizon"])
def test_graph_replays_equal_eager_updates(kw):
    mem_kw = dict(TRUNC, **{k: v for k, v in kw.items() if k in ("anneal_steps", "multi_step_start", "discount_start",
                                                                 "multi_step", "discount")})
    ga, gm = _agent(**TRUNC, **kw), _memory(**mem_kw)
    ea, em = _agent(cuda_graph=False, **TRUNC, **kw), _memory(**mem_kw)
    for _ in range(6):
        for ag, mem in ((ga, gm), (ea, em)):
            ag.reset_noise()
            ag.learn(mem)
    assert ga._graphs and not ea._graphs
    _assert_snapshots(_snapshot(ga, gm), _snapshot(ea, em), "graph vs eager")
    assert np.isfinite(cpu(ga.last_loss)).all()


def test_switches_must_agree():
    from rainbow_b200._lib import RainbowB200Error
    with pytest.raises(RainbowB200Error, match="bootstrap_truncation"):
        _agent(**TRUNC).learn(_memory())
    with pytest.raises(RainbowB200Error, match="bootstrap_truncation"):
        _agent().learn(_memory(**TRUNC))


@pytest.mark.parametrize("batch", [32, 64])
def test_update_graph_swaps_only_the_gather(batch, tmp_path, monkeypatch):
    plain = update_graph(_agent(batch_size=batch), _memory(), tmp_path / "plain.dot", monkeypatch)
    on = update_graph(_agent(batch_size=batch, **TRUNC), _memory(**TRUNC), tmp_path / "on.dot", monkeypatch)
    assert len(on) == len(plain)
    assert on.count("k_gather_hz_trunc") == plain.count("k_gather") == 1
    assert [("k_gather" if k == "k_gather_hz_trunc" else k) for k in on] == plain


def test_resume_with_final_observations_equals_never_stopping(tmp_path):
    import json
    from rainbow_b200._lib import RainbowB200Error
    from rainbow_b200.memory import ReplayMemory

    def run(ag, mem, steps, losses):
        for _ in steps:
            ag.reset_noise()
            ag.learn(mem)
            losses.append(ag.last_loss.clone())

    ag, mem = _agent(**TRUNC), _memory(**TRUNC)
    la = []
    run(ag, mem, range(8), la)
    a = dict(_snapshot(ag, mem), losses=cpu(torch.stack(la)))
    ag, mem = _agent(**TRUNC), _memory(**TRUNC)
    lb = []
    run(ag, mem, range(3), lb)
    ag.save_checkpoint(str(tmp_path / "ck"), mem)
    man = json.load(open(tmp_path / "ck" / "rank0" / "manifest.json"))
    assert man["hyper_parameters"]["bootstrap_truncation"] is True and man["replay"]["final_records"] is True
    plain_mem = ReplayMemory(make_args(), CAP, seed=12345)
    before = cpu(plain_mem.transitions.nonterminal).copy()
    with pytest.raises(RainbowB200Error, match="final-observation records"):
        _agent(seed=77).load_checkpoint(str(tmp_path / "ck"), plain_mem)
    assert_bits_equal(cpu(plain_mem.transitions.nonterminal), before, "a refused load wrote the ring")
    ag, mem = _agent(seed=77, **TRUNC), ReplayMemory(make_args(**TRUNC), CAP, seed=12345)
    ag.load_checkpoint(str(tmp_path / "ck"), mem)
    run(ag, mem, range(3, 8), lb)
    b = dict(_snapshot(ag, mem), losses=cpu(torch.stack(lb)))
    _assert_snapshots(a, b, "resumed vs uninterrupted")
