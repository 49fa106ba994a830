"""Polyak target updates (rb_target_ema, args.target_tau) and shrink-and-perturb resets (rb_param_reset,
Agent.reset_parameters, args.reset_interval) on the GPU.

* rb_target_ema: bitwise the numpy fp32 blend of tests/reset_ref.py (exact fma) for n = 1 ... 6.9 M around the grid-stride
  wrap, n % 4 != 0 and either pointer misaligned, tau = 1e-3 / 0.005 / 0.5 / 1 (1 is a copy); a gate reading 0 writes
  nothing; guard elements stay untouched; a graph replay equals the eager launch.
* The learner with tau > 0: after every eager update the target equals the blend of the target before it and the online
  parameters after it, bitwise (fused head with the draw pending and flushed, batch 64, C3, the library head, shift 4 with
  M = K = 2); seven graph replays equal seven eager updates; tau = 1 is an agent calling update_target_net() after every
  learn(); a rejected batch leaves the target alone; the update graph is the graph without the option plus one
  k_target_ema right after k_clip_adam.
* rb_param_reset: bitwise the numpy theta0 and blend for alpha = 0 / 0.5 / 0.8 / 1 (1 a no-op); padding, guards, elements
  outside every segment, the Adam state, the target, the noise and the replay untouched; successive resets draw afresh;
  over the canonical net each uniform tensor lies in [-b, b) and passes a KS test, sigma equals its constant; a graph
  replayed after a reset equals an eager update from the same state.
* Schedule and resume: reset_interval fires after the N-th, 2N-th, ... learn(); 5 updates + save + load + 7 equal 12
  uninterrupted ones (tau 0.005, interval 4, shrink_encoder 0.5, data-efficient / 256, shift 4); a manifest without the
  new keys loads.  Two ranks stay bitwise identical through updates and a reset.
Deterministic cuDNN, like the other trajectory tests."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import reset_ref as R
from helpers import assert_bits_equal
from test_gpu_augment import GUARD, update_graph
from test_gpu_parity import DEV, FakeEnv, cpu, make_args, synthetic_ring

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAP = 8192


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


# ---- rb_target_ema ---------------------------------------------------------------------------------------------------------
WRAP = 132 * 8 * 256 * 4        # elements one float4 sweep of the largest grid covers
SIZES = [1, 2, 3, 4, 5, 7, 8, 1023, 4097, WRAP - 1, WRAP, WRAP + 3, 2 * WRAP + 5, 6_900_003]
TAUS = [1e-3, 0.005, 0.5, 1.0]
OFFSETS = [(0, 0), (1, 0), (0, 3)]
EMA_CASES = [(n, tau, OFFSETS[(i + j) % 3]) for i, n in enumerate(SIZES) for j, tau in enumerate(TAUS)
             if n < 2 * WRAP or tau in (0.005, 1.0)]


def ema_launch(target, param, n, tau, gate=None, ot=0, op=0):
    rc = lib().rb_target_ema(target.data_ptr() + 4 * ot, param.data_ptr() + 4 * op, n, tau,
                             None if gate is None else gate.data_ptr(), stream())
    assert rc == 0, lib().rb_last_error()


def ema_buffers(n, ot, op, seed):
    rs = np.random.RandomState(seed)
    t0 = rs.randn(ot + n + GUARD).astype(np.float32)
    p0 = rs.randn(op + n + GUARD).astype(np.float32)
    return t0, p0, torch.from_numpy(t0).to(DEV), torch.from_numpy(p0).to(DEV)


@pytest.mark.parametrize("n,tau,offs", EMA_CASES, ids=[f"n{n}-tau{t}-off{o[0]}{o[1]}" for n, t, o in EMA_CASES])
def test_target_ema_is_the_fp32_blend(n, tau, offs):
    ot, op = offs
    t0, p0, T, Pd = ema_buffers(n, ot, op, n % 9973 + int(tau * 1000))
    ema_launch(T, Pd, n, tau, ot=ot, op=op)
    got = cpu(T)
    want = R.ema_ref(t0[ot:ot + n], p0[op:op + n], tau)
    assert_bits_equal(got[ot:ot + n], want, f"n={n} tau={tau}")
    assert_bits_equal(got[:ot], t0[:ot], "elements before the target")
    assert_bits_equal(got[ot + n:], t0[ot + n:], "guard elements past n")
    assert_bits_equal(cpu(Pd), p0, "param is read only")
    if tau == 1.0:
        assert_bits_equal(got[ot:ot + n], p0[op:op + n], "tau = 1 copies")


@pytest.mark.parametrize("n", [4097, 1_000_003])
def test_target_ema_gate_and_graph_replay(n):
    t0, p0, T, Pd = ema_buffers(n, 0, 0, 17)
    gate = torch.zeros(1, dtype=torch.int32, device=DEV)
    ema_launch(T, Pd, n, 0.005, gate=gate)
    assert_bits_equal(cpu(T), t0, "a gate reading 0 writes nothing")
    gate.fill_(1)
    ema_launch(T, Pd, n, 0.005, gate=gate)
    eager = cpu(T).copy()
    assert_bits_equal(eager[:n], R.ema_ref(t0[:n], p0[:n], 0.005), "gate 1 = no gate")
    T.copy_(torch.from_numpy(t0))
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            ema_launch(T, Pd, n, 0.005, gate=gate)
    assert_bits_equal(cpu(T), t0, "capturing does not execute")
    g.replay()
    assert_bits_equal(cpu(T), eager, "graph replay == eager launch")


# ---- the learner with tau > 0 ----------------------------------------------------------------------------------------------
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


C3 = dict(architecture="data-efficient", hidden_size=256)
LEARNER_CASES = {
    "fused-pending": (dict(), True),
    "fused-flushed": (dict(), False),
    "batch64-large-backward": (dict(batch_size=64), True),
    "c3": (C3, True),
    "library-head": (dict(fused_head=False), False),
    "c3-shift4-m2-k2": (dict(augment_shift=4, augment_m=2, augment_k=2, **C3), True),
}


@pytest.mark.parametrize("case", list(LEARNER_CASES))
def test_learner_target_is_the_blend_after_every_update(case):
    kw, pending = LEARNER_CASES[case]
    tau = 0.005
    ag, mem = _agent(target_tau=tau, cuda_graph=False, **kw), _memory()
    assert ag._fused_path(ag.batch_size) == (case != "library-head")
    if case.startswith("batch64"):
        assert ag.batch_size > 32    # k_head_bwd1's limit: the large-batch layer-1 kernels run
    base, end = ag.target_flat.data_ptr(), ag.target_flat.data_ptr() + 4 * ag.target_flat.numel()
    assert all(base <= p.data_ptr() < end for p in ag.target_net.parameters()), "the target's parameters are views"
    ag.target_flat.mul_(0.5)         # target != online, so that tau and 1 - tau cannot be confused unnoticed
    for step in range(3):
        ag.reset_noise()
        if not pending:
            ag.online_net.flush_noise()
        t0 = cpu(ag.target_flat).copy()
        ag.learn(mem)
        torch.cuda.synchronize()
        assert int(ag.optimiser.step_count.item()) == step + 1
        want = R.ema_ref(t0, cpu(ag.optimiser.flat_param), tau)
        assert_bits_equal(cpu(ag.target_flat), want, f"target after update {step}")
    assert (cpu(ag.target_flat) != t0).any()


def test_graph_replay_equals_eager():
    ga, ea = _agent(target_tau=0.005), _agent(target_tau=0.005, cuda_graph=False)
    gm, em = _memory(), _memory()
    for step in range(7):
        for ag, mem in ((ga, gm), (ea, em)):
            ag.reset_noise()
            ag.learn(mem)
        assert_bits_equal(cpu(ga.last_loss), cpu(ea.last_loss), f"loss of update {step}")
    assert ga._graphs and not ea._graphs
    _assert_snapshots(_snapshot(ga, gm), _snapshot(ea, em), "graph vs eager")


def test_tau_one_is_a_hard_copy_after_every_learn():
    soft, hard = _agent(target_tau=1.0, cuda_graph=False), _agent(cuda_graph=False)
    ms, mh = _memory(), _memory()
    for step in range(4):
        soft.reset_noise()
        soft.learn(ms)
        hard.reset_noise()
        hard.learn(mh)
        hard.update_target_net()
        assert_bits_equal(cpu(soft.last_loss), cpu(hard.last_loss), f"loss of update {step}")
        _assert_snapshots(_snapshot(soft, ms), _snapshot(hard, mh), f"after update {step}")
        assert_bits_equal(cpu(soft.target_flat), cpu(soft.optimiser.flat_param), "tau = 1: target == online")


@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
def test_rejected_batch_leaves_the_target(use_graph):
    """The setup of test_rejected_batch_is_skipped_on_device: every draw fails, the batch is rejected, the step skipped."""
    from rainbow_b200.agent import Agent
    from rainbow_b200.memory import ReplayMemory
    torch.manual_seed(1)
    args = make_args(cuda_graph=use_graph, architecture="data-efficient", hidden_size=64, batch_size=8, target_tau=0.5)
    mem = ReplayMemory(args, 256, max_attempts=3, seed=4)
    tr = mem.transitions
    tr.load_arrays(timestep=np.arange(256) % 50, action=np.zeros(256), reward=np.ones(256), nonterminal=np.ones(256), index=10,
                   full=True, t_episode=11)
    tr.frames.fill_(7)
    ag = Agent(args, FakeEnv(4))
    ag.target_flat.mul_(0.5)
    t0 = cpu(ag.target_flat).copy()
    for _ in range(5):
        ag.reset_noise()
        ag.learn(mem)
    torch.cuda.synchronize()
    assert int(ag.optimiser.step_count.item()) == 0
    assert_bits_equal(cpu(ag.target_flat), t0, "a rejected batch moves the target")
    tr.update(np.arange(256) + tr.tree_start, np.full(256, 0.5, np.float32))
    ag.reset_noise()
    ag.learn(mem)
    torch.cuda.synchronize()
    assert int(ag.optimiser.step_count.item()) == 1
    assert_bits_equal(cpu(ag.target_flat), R.ema_ref(t0, cpu(ag.optimiser.flat_param), 0.5), "the applied step's blend")


@pytest.mark.parametrize("batch", [32, 64])
def test_update_graph_adds_one_node_after_clip_adam(batch, tmp_path, monkeypatch):
    names = {}
    for tag, kw in (("default", dict()), ("zero", dict(target_tau=0.0)), ("on", dict(target_tau=0.005))):
        names[tag] = update_graph(_agent(batch_size=batch, **kw), _memory(), tmp_path / f"{tag}.dot", monkeypatch)
    assert names["zero"] == names["default"], "target_tau = 0 leaves the update graph as it is"
    on = names["on"]
    assert on.count("k_target_ema") == 1 and "k_target_ema" not in names["default"]
    i = on.index("k_target_ema")
    assert on[i - 1] == "k_clip_adam", on[i - 3:i + 2]
    assert on[:i] + on[i + 1:] == names["default"]


# ---- rb_param_reset --------------------------------------------------------------------------------------------------------
def _table(ag, alphas):
    from rainbow_b200.agent import reset_table
    return [(o, n, b, c, alphas[g]) for o, n, b, c, g in reset_table(ag.online_net, ag.optimiser.offsets)]


def reset_launch(buf, n, segs, seed, k):
    from rainbow_b200 import _lib
    arr = (_lib.ResetSegment * len(segs))(*[_lib.ResetSegment(*s) for s in segs])
    rc = lib().rb_param_reset(buf.data_ptr(), n, arr, len(segs), seed, k, stream())
    assert rc == 0, lib().rb_last_error()


@pytest.mark.parametrize("alpha", [0.0, 0.5, 0.8, 1.0])
def test_param_reset_is_the_numpy_draw_and_blend(alpha):
    ag = _agent(cuda_graph=False)
    segs = _table(ag, (alpha, alpha))
    numel = ag.optimiser.numel
    rs = np.random.RandomState(int(alpha * 10))
    p0 = rs.randn(numel + GUARD).astype(np.float32)
    buf = torch.from_numpy(p0).to(DEV)
    seed, k = 0x0123456789ABCDEF, (1 << 32) + 3
    reset_launch(buf, numel, segs, seed, k)
    got = cpu(buf)
    want, drawn = R.reset_ref(p0[:numel], segs, seed, k)
    assert_bits_equal(got[:numel], want, f"alpha {alpha}")
    assert_bits_equal(got[numel:], p0[numel:], "guard elements")
    covered = np.zeros(numel, bool)
    for o, n, *_ in segs:
        covered[o:o + n] = True
    assert (~covered).sum() > 0 and np.array_equal(got[:numel][~covered], p0[:numel][~covered]), "padding is written"
    if alpha == 1.0:
        assert_bits_equal(got, p0, "alpha = 1 is a no-op")
    if alpha == 0.0:
        assert_bits_equal(got[:numel][covered], np.concatenate(drawn), "alpha = 0 is theta0")


def test_param_reset_segments_off_the_quad_grid():
    """Segments that start and end inside a Philox quad: the elements of the quad outside them stay as they were."""
    segs = [(3, 10, 0.2, 0.0, 0.0), (13, 1, 0.0, 0.3, 0.0), (14, 2, 0.5, 0.0, 0.25), (21, 5, 0.1, 0.0, 0.5),
            (40, 24, 0.0, 0.01, 0.75)]
    p0 = np.random.RandomState(2).randn(64 + GUARD).astype(np.float32)
    buf = torch.from_numpy(p0).to(DEV)
    reset_launch(buf, 64, segs, 5, 9)
    assert_bits_equal(cpu(buf)[:64], R.reset_ref(p0[:64], segs, 5, 9)[0], "quad-straddling segments")
    assert_bits_equal(cpu(buf)[64:], p0[64:], "guards")


def test_reset_parameters_touches_only_the_online_parameters():
    ag, mem = _agent(cuda_graph=False), _memory()
    for _ in range(2):
        ag.reset_noise()
        ag.learn(mem)
    ag.reset_noise()
    torch.cuda.synchronize()
    on, tg, o = ag.online_net, ag.target_net, ag.optimiser

    def rest():
        d = dict(exp_avg=o.exp_avg, exp_avg_sq=o.exp_avg_sq, step=o.step_count, target=ag.target_flat, tree=mem.transitions.tree,
                 rng=mem._rng_counter)
        for tag, net in (("online", on), ("target", tg)):
            d.update({f"{tag}.counter": net._noise_counter, f"{tag}.f_in": net._f_in, f"{tag}.f_out": net._f_out})
            d.update((f"{tag}.{n}", b) for n, b in net.named_buffers() if n.endswith("_epsilon"))
        torch.cuda.synchronize()
        return {k: cpu(v).copy() for k, v in d.items()}

    before, p0 = rest(), cpu(o.flat_param).copy()
    pending = on._noise_pending
    ag.reset_parameters(0.5, 0.0)
    torch.cuda.synchronize()
    assert ag.reset_count == 1 and on._noise_pending == pending
    want, drawn0 = R.reset_ref(p0, _table(ag, (0.5, 0.0)), ag.reset_seed, 0)
    assert_bits_equal(cpu(o.flat_param), want, "shrink 0.5 encoder, re-initialised head")
    after = rest()
    for k in before:
        assert_bits_equal(after[k], before[k], f"{k} is untouched by a reset")
    ag.reset_parameters()
    torch.cuda.synchronize()
    want1, drawn1 = R.reset_ref(want, _table(ag, (1.0, 0.0)), ag.reset_seed, 1)
    assert_bits_equal(cpu(o.flat_param), want1, "the second reset draws with index 1")
    conv = sum(1 for s in _table(ag, (0, 1)) if s[4] == 0)
    for a, b, s in zip(drawn0, drawn1, _table(ag, (0.0, 0.0))):
        if s[2] > 0:
            assert not np.array_equal(a, b), "successive resets draw different theta0"
    assert conv == 6
    with pytest.raises(ValueError):
        ag.reset_parameters(1.5, 0.0)
    with pytest.raises(ValueError):
        ag.reset_parameters(1.0, float("nan"))
    assert ag.reset_count == 2


def test_fresh_draws_follow_the_initialisation():
    """Each re-drawn tensor against its table entry (range, KS against U[-b, b), sigma constants exactly) and against the
    tensor torch's own Conv2d / NoisyLinear initialisation draws for a fresh module of that shape (two-sample KS)."""
    from scipy import stats
    from torch import nn

    from rainbow_b200.model import NoisyLinear
    ag = _agent(cuda_graph=False)
    ag.reset_parameters(0.0, 0.0)
    torch.cuda.synchronize()
    flat = cpu(ag.optimiser.flat_param)
    for (o, n, b, c, _), (name, _) in zip(_table(ag, (0.0, 0.0)), ag.online_net.named_parameters()):
        v = flat[o:o + n]
        owner, kind = name.rsplit(".", 1)
        m = ag.online_net.get_submodule(owner)
        if isinstance(m, nn.Conv2d):
            fresh = nn.Conv2d(m.in_channels, m.out_channels, m.kernel_size, stride=m.stride)
        else:
            fresh = NoisyLinear(m.in_features, m.out_features, std_init=m.std_init)
        ref = getattr(fresh, kind).detach().numpy().ravel()
        if b == 0.0:
            assert (v == np.float32(c)).all() and (ref == np.float32(c)).all(), name
            continue
        bb = np.float32(b)
        assert v.min() >= -bb and v.max() < bb, name
        assert stats.kstest(v.astype(np.float64), stats.uniform(loc=-b, scale=2 * b).cdf).pvalue > 1e-4, name
        if n >= 1000:
            assert stats.ks_2samp(v, ref).pvalue > 1e-4, f"{name}: theta0 is not distributed as torch initialises it"


def test_graph_after_a_reset_equals_eager():
    ga, ea = _agent(target_tau=0.005), _agent(target_tau=0.005, cuda_graph=False)
    gm, em = _memory(), _memory()
    for step in range(6):
        for ag, mem in ((ga, gm), (ea, em)):
            ag.reset_noise()
            ag.learn(mem)
            if step == 3:
                ag.reset_parameters(0.5, 0.0)
        assert_bits_equal(cpu(ga.last_loss), cpu(ea.last_loss), f"loss of update {step}")
        _assert_snapshots(_snapshot(ga, gm), _snapshot(ea, em), f"after update {step}")
    assert ga._graphs and ga.reset_count == ea.reset_count == 1


# ---- schedule and resume ---------------------------------------------------------------------------------------------------
def test_reset_interval_fires_after_every_nth_learn(monkeypatch):
    ag, mem = _agent(reset_interval=3, reset_shrink_encoder=0.25, architecture="data-efficient", hidden_size=64), _memory()
    calls, orig = [], ag.reset_parameters

    def spy(*a):
        calls.append((ag._learn_calls, a))
        return orig(*a)

    monkeypatch.setattr(ag, "reset_parameters", spy)
    for _ in range(10):
        ag.reset_noise()
        ag.learn(mem)
    assert calls == [(3, (0.25, 0.0)), (6, (0.25, 0.0)), (9, (0.25, 0.0))]
    assert ag.reset_count == 3
    for bad in (dict(target_tau=1.5), dict(reset_interval=-2), dict(reset_shrink_head=-0.1)):
        with pytest.raises(ValueError):
            _agent(architecture="data-efficient", hidden_size=64, **bad)


def test_resume_equals_never_stopping(tmp_path):
    """tau 0.005, a reset every 4 updates (encoder shrunk by 0.5), data-efficient / 256 with shift 4: 5 updates, save, fresh
    objects, load, 7 more == 12 uninterrupted updates, bitwise.  Resets fall after updates 4 (before the save), 8 and 12."""
    from test_gpu_checkpoint import _agent as ck_agent
    from test_gpu_checkpoint import _assert_same, _before_update, _fresh_memory, _state, _update
    from test_gpu_checkpoint import _memory as ck_memory
    kw = dict(target_tau=0.005, reset_interval=4, reset_shrink_encoder=0.5, augment_shift=4, **C3)
    total, save_at = 12, 5
    ag, mem = ck_agent(**kw), ck_memory()
    losses = []
    for step in range(total):
        _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    run_a = _state(ag, mem, losses)
    assert ag.reset_count == 3

    ag, mem = ck_agent(**kw), ck_memory()
    losses = []
    for step in range(save_at):
        _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _before_update(ag, mem, save_at, True)
    ag.save_checkpoint(str(tmp_path / "ck"), mem)
    man = json.load(open(tmp_path / "ck" / "rank0" / "manifest.json"))
    hp, learner = man["hyper_parameters"], man["learner"]
    assert (hp["target_tau"], hp["reset_interval"], hp["reset_shrink_encoder"]) == (0.005, 4, 0.5)
    assert "reset_shrink_head" not in hp
    assert (learner["reset_seed"], learner["reset_count"]) == (ag.reset_seed, 1)
    ag, mem = ck_agent(seed=77, **kw), _fresh_memory()
    assert ag.reset_count == 0
    ag.load_checkpoint(str(tmp_path / "ck"), mem)
    assert ag.reset_count == 1 and ag.reset_seed == learner["reset_seed"]
    for step in range(save_at, total):
        if step > save_at:
            _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _assert_same(run_a, _state(ag, mem, losses))
    assert ag.reset_count == 3


def test_resume_saved_before_the_first_reset_under_another_torch_seed(tmp_path):
    """A checkpoint taken before any reset still carries the reset key: 3 updates, save, fresh objects under another torch
    seed (so another live key), load, 6 more == 9 uninterrupted updates, bitwise, with resets after updates 4 and 8."""
    from test_gpu_checkpoint import _agent as ck_agent
    from test_gpu_checkpoint import _assert_same, _before_update, _fresh_memory, _state, _update
    from test_gpu_checkpoint import _memory as ck_memory
    kw = dict(reset_interval=4, reset_shrink_encoder=0.5, architecture="data-efficient", hidden_size=64)
    total, save_at = 9, 3
    ag, mem = ck_agent(**kw), ck_memory()
    losses = []
    for step in range(total):
        _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    run_a = _state(ag, mem, losses)
    assert ag.reset_count == 2

    ag, mem = ck_agent(**kw), ck_memory()
    losses = []
    for step in range(save_at):
        _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _before_update(ag, mem, save_at, True)
    ag.save_checkpoint(str(tmp_path / "ck"), mem)
    learner = json.load(open(tmp_path / "ck" / "rank0" / "manifest.json"))["learner"]
    assert (learner["reset_seed"], learner["reset_count"]) == (ag.reset_seed, 0)
    saved_seed = ag.reset_seed
    ag, mem = ck_agent(seed=99, **kw), _fresh_memory()
    assert ag.reset_seed != saved_seed, "the resumed process has another live key"
    ag.load_checkpoint(str(tmp_path / "ck"), mem)
    assert ag.reset_seed == saved_seed and ag.reset_count == 0
    for step in range(save_at, total):
        if step > save_at:
            _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _assert_same(run_a, _state(ag, mem, losses))
    assert ag.reset_count == 2


def test_manifest_without_the_new_keys_loads(tmp_path):
    """Runs with both options off write the manifest of before plus the reset key and count; a manifest from before those
    keys existed (here: the keys taken out and the digest recomputed) loads as no reset yet, with the live key."""
    from rainbow_b200 import checkpoint as ckpt
    from test_gpu_checkpoint import _agent as ck_agent
    plain = ck_agent()
    plain.save_checkpoint(str(tmp_path / "plain"))
    path = tmp_path / "plain" / "rank0" / "manifest.json"
    man = json.load(open(path))
    for k in ("target_tau", "reset_interval", "reset_shrink_encoder", "reset_shrink_head"):
        assert k not in man["hyper_parameters"], k
    assert (man["learner"]["reset_seed"], man["learner"]["reset_count"]) == (plain.reset_seed, 0)
    del man["learner"]["reset_seed"], man["learner"]["reset_count"]
    man["digest"] = ckpt._digest(man)
    json.dump(man, open(path, "w"), indent=1, sort_keys=True)
    ag = ck_agent(seed=9, target_tau=0.005, reset_interval=4)
    live_seed = ag.reset_seed
    ag.reset_parameters()
    assert ag.reset_count == 1
    ag.load_checkpoint(str(tmp_path / "plain"))
    assert ag.reset_count == 0 and ag.reset_seed == live_seed, "absent = no reset yet, with the live key"
    assert_bits_equal(cpu(ag.optimiser.flat_param), cpu(plain.optimiser.flat_param), "parameters")
    assert_bits_equal(cpu(ag.target_flat), cpu(plain.target_flat), "target (through the target.* views)")
    # one of the pair without the other is refused, and the refusal changes nothing
    man["learner"]["reset_count"] = 3
    man["digest"] = ckpt._digest(man)
    json.dump(man, open(path, "w"), indent=1, sort_keys=True)
    ag.reset_parameters()
    with pytest.raises(Exception, match="together"):
        ag.load_checkpoint(str(tmp_path / "plain"))
    assert ag.reset_count == 1 and ag.reset_seed == live_seed


# ---- two ranks -------------------------------------------------------------------------------------------------------------
_DP_WORKER = r"""
import os, sys
import torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
from rainbow_b200.dist import init_from_env
ngpu = torch.cuda.device_count()
backend = "nccl" if ngpu >= 2 else "gloo"          # one GPU: both ranks share it, gloo moves the CUDA tensors
if backend == "gloo":
    os.environ["LOCAL_RANK"] = "0"
rank, world, local = init_from_env(backend)
from test_gpu_parity import FakeEnv, make_args, synthetic_ring
from rainbow_b200.agent import Agent
dev = torch.device("cuda", local)
torch.cuda.set_device(dev)
def same_everywhere(x, what):
    a = x.detach().to(dev, torch.float64)
    lo, hi = a.clone(), a.clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN); dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    assert torch.equal(lo, hi), what
torch.manual_seed(7)
args = make_args(device=dev, cuda_graph=False, architecture="data-efficient", hidden_size=64, batch_size=8, target_tau=0.005,
                 reset_interval=3, reset_shrink_encoder=0.5, peer_optimizer="auto" if backend == "nccl" else False)
mem, _ = synthetic_ring(1024, seed=10, device=str(dev), args=dict(device=dev))
torch.manual_seed(100 + rank)                       # a different torch seed per rank: the reset key must still agree
ag = Agent(args, FakeEnv(4))
same_everywhere(torch.tensor([ag.reset_seed >> 32, ag.reset_seed & 0xFFFFFFFF]), "reset seeds differ across ranks")
for step in range(5):
    ag.reset_noise(); ag.learn(mem)
    torch.cuda.synchronize()
    same_everywhere(ag.optimiser.flat_param, f"parameters diverged after update {step}")
    same_everywhere(ag.target_flat, f"targets diverged after update {step}")
assert ag.reset_count == 1 and int(ag.optimiser.step_count.item()) == 5
ag.reset_parameters(0.5, 0.2)
torch.cuda.synchronize()
same_everywhere(ag.optimiser.flat_param, "parameters diverged after a reset")
ag.reset_noise(); ag.learn(mem)
torch.cuda.synchronize()
same_everywhere(ag.optimiser.flat_param, "parameters diverged after the update that followed a reset")
same_everywhere(ag.target_flat, "targets diverged after the update that followed a reset")
dist.barrier()
dist.destroy_process_group()
print(f"rank{rank}ok backend={backend} peer={ag.peer_optimizer}", flush=True)
"""


def test_two_ranks_stay_identical_through_updates_and_resets(tmp_path):
    script = tmp_path / "dp_target_reset.py"
    script.write_text(_DP_WORKER)
    port = 29500 + os.getpid() % 190
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(script), ROOT]
    env = dict(os.environ, OMP_NUM_THREADS="1")
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-4000:]
    assert out.stdout.count("ok backend=") == 2, out.stdout
