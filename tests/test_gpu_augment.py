"""Random-shift augmentation of the sampled states (rb_gather_shift / ReplayMemory.sample_into(ws, shift_pad) /
args.augment_shift) on the GPU.

* The kernel: states and next states equal the numpy shift (tests/philox_ref.py: edge pad, then crop) of rb_gather's own
  output at the recorded offsets, bitwise; the scalar outputs equal rb_gather's; guard rows stay untouched; a graph replay
  equals the eager launch; the graph's node is k_gather_shift.  Over history / n 4/3, 4/20, 4/1, 1/1, 4/60, episode
  boundaries inside the window, index wrap, split 1 and 2, B 1 ... 2048 and pad 1 / 4 / 16.
* The draws: the recorded offsets are philox_ref's for the replay's seed and counter; over 10^5 samples every cell occurs,
  the cells are uniform (chi-square), state and next-state offsets are independent, and successive batches differ.
* The learner: augmented updates equal a twin agent's unaugmented updates fed the same batch shifted in numpy, bitwise, at
  C2 / C3 shapes and batch 64 (the large-batch layer-1 backward); graph replay equals eager; the update graph is the one without
  augmentation with k_gather replaced by k_gather_shift; a checkpointed run resumes bitwise.
* The surface: acting and evaluation are unaugmented, rng="numpy" and a foreign memory are refused, and augment_shift = 0
  leaves the update graph as it was.
Like the other trajectory tests this one runs with deterministic cuDNN algorithms (DESIGN.md §9)."""
import functools
import html
import json
import re

import numpy as np
import pytest
import torch

import philox_ref as P
from helpers import assert_bits_equal
from test_gpu_parity import DEV, FakeEnv, cpu, make_args, synthetic_ring

pytestmark = pytest.mark.gpu

CAP = 8192
GUARD = 2
NAN = float("nan")


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


def episodic_memory(history, n, cap=4096, seed=0):
    """synthetic_ring with episodes of 2 ... 70 steps, so most windows (up to 64 records) hold an episode boundary."""
    mem, _ = synthetic_ring(cap, seed=seed, args=dict(history_length=history, multi_step=n))
    rs = np.random.RandomState(seed + 1)
    ts = []
    while len(ts) < cap:
        ts.extend(range(rs.randint(2, 71)))
    ts = np.array(ts[:cap], dtype=np.int32)
    mem.transitions.timestep.copy_(torch.from_numpy(ts))
    return mem, ts


class Outputs:
    """The buffers one gather writes, each with GUARD rows past the batch, prefilled with NaN / -1 / -7."""

    def __init__(self, B, history):
        self.B = B
        self.states = torch.full((B + GUARD, history, 84, 84), NAN, device=DEV)
        self.next_states = torch.full((B + GUARD, history, 84, 84), NAN, device=DEV)
        self.actions = torch.full((B + GUARD,), -1, dtype=torch.int64, device=DEV)
        self.returns = torch.full((B + GUARD,), NAN, device=DEV)
        self.nonterminals = torch.full((B + GUARD,), NAN, device=DEV)
        self.shifts_flat = torch.full((4 * B + 8,), -7, dtype=torch.int32, device=DEV)
        self.shifts = self.shifts_flat[:4 * B].view(2, B, 2)

    def host(self):
        B = self.B
        return dict(states=cpu(self.states[:B]), next_states=cpu(self.next_states[:B]), actions=cpu(self.actions[:B]),
                    returns=cpu(self.returns[:B]), nonterminals=cpu(self.nonterminals[:B]), shifts=cpu(self.shifts))

    def assert_guards(self):
        B = self.B
        assert torch.isnan(self.states[B:]).all() and torch.isnan(self.next_states[B:]).all()
        assert (self.actions[B:] == -1).all() and torch.isnan(self.returns[B:]).all()
        assert torch.isnan(self.nonterminals[B:]).all() and (self.shifts_flat[4 * B:] == -7).all()


def gather(mem, didx, out, pad=0, seed=0, counter=None):
    tr = mem.transitions
    p = lambda t: t.data_ptr()
    common = (p(tr.frames), p(tr.timestep), p(tr.action), p(tr.reward), p(tr.nonterminal), tr.size, p(didx), out.B,
              mem.history, mem.n, p(mem.n_step_scaling), p(out.states), p(out.next_states), p(out.actions), p(out.returns),
              p(out.nonterminals))
    if pad == 0:
        rc = lib().rb_gather(*common, stream())
    else:
        rc = lib().rb_gather_shift(*common, pad, seed, p(counter), p(out.shifts), stream())
    assert rc == 0, lib().rb_last_error()


# (history, n, B, pad)
KERNEL_CASES = [(4, 3, 32, 4), (4, 3, 32, 1), (4, 3, 32, 16), (4, 20, 32, 4), (4, 1, 32, 16), (1, 1, 32, 4), (4, 60, 32, 1),
                (4, 3, 1, 16), (4, 60, 1, 4), (4, 3, 512, 4), (1, 1, 512, 16), (4, 20, 512, 1), (4, 3, 2048, 4),
                (4, 60, 2048, 16)]


@pytest.mark.parametrize("history,n,B,pad", KERNEL_CASES, ids=[f"h{h}-n{n}-B{B}-p{p}" for h, n, B, p in KERNEL_CASES])
def test_kernel_is_the_numpy_shift_of_rb_gather(history, n, B, pad, tmp_path):
    from test_gpu_head_f64 import graph_kernels
    mem, ts = episodic_memory(history, n)
    cap = mem.capacity
    rs = np.random.RandomState(B * 131 + pad * 7 + history + n)
    idx = rs.randint(0, cap, B)
    idx[:min(B, 4)] = [0, 1, cap - 1, 2][:min(B, 4)]               # windows that wrap around the ring's ends
    idx[4:8] = rs.choice(np.flatnonzero(ts == 1), 4)[:max(0, min(B, 8) - 4)]   # the state's oldest frames blanked
    didx = torch.from_numpy(idx.astype(np.int64)).to(DEV)
    seed = int(rs.randint(0, 2 ** 62)) * 3 + 1
    c = (int(rs.randint(1, 2 ** 20)) << 32) + int(rs.randint(0, 2 ** 31))
    counter = torch.tensor([c], dtype=torch.int64, device=DEV)

    plain, shifted = Outputs(B, history), Outputs(B, history)
    gather(mem, didx, plain)
    gather(mem, didx, shifted, pad, seed, counter)
    torch.cuda.synchronize()
    a, s = plain.host(), shifted.host()
    plain.assert_guards()
    shifted.assert_guards()
    assert int(counter.item()) == c, "the gather reads the counter, it does not advance it"

    want = P.shift_offsets(seed, c, B, pad)
    assert_bits_equal(s["shifts"], want, "offsets")
    assert want.min() >= 0 and want.max() <= 2 * pad
    assert_bits_equal(s["states"], P.shift_ref(a["states"], want[0], pad), "states")
    assert_bits_equal(s["next_states"], P.shift_ref(a["next_states"], want[1], pad), "next_states")
    for k in ("actions", "returns", "nonterminals"):
        assert_bits_equal(s[k], a[k], k)
    # the case exercises what it claims: blanked frames inside windows, and samples moved off the identity
    assert (a["states"].reshape(B, history, -1).max(axis=2) == 0).any() or B == 1 or history == 1
    assert (want != pad).any()

    replay = Outputs(B, history)
    _, _, dot = graph_kernels(lambda: gather(mem, didx, replay, pad, seed, counter), tmp_path / "gather.dot")
    assert "k_gather_shift" in dot
    r = replay.host()
    for k in s:
        assert_bits_equal(r[k], s[k], "graph replay: " + k)
    replay.assert_guards()


@pytest.mark.parametrize("pad", [1, 4, 16])
def test_draws_follow_the_philox_stream_and_are_uniform(pad):
    from rainbow_b200.memory import _SampleWorkspace
    from scipy import stats
    mem, _ = synthetic_ring(65536, seed=2)
    mem.seed = 0x9E3779B97F4A7C15
    B, rounds = 2048, 50
    ws = _SampleWorkspace(B, mem.history, mem.device)
    offs, prev = [], None
    for _ in range(rounds):
        mem.sample_into(ws, shift_pad=pad)
        sh = cpu(ws.shifts).copy()
        c = int(mem._rng_counter.item())
        assert_bits_equal(sh, P.shift_offsets(mem.seed, c, B, pad), f"offsets at counter {c}")
        assert prev is None or not np.array_equal(sh, prev), "successive batches draw afresh"
        prev = sh
        offs.append(sh)
    offs = np.concatenate(offs, axis=1)                      # [2][rounds * B][2]
    k = 2 * pad + 1
    for side in (0, 1):
        cells = np.bincount(offs[side, :, 0] * k + offs[side, :, 1], minlength=k * k)
        assert cells.size == k * k and (cells > 0).all(), "every (oy, ox) occurs"
        assert stats.chisquare(cells).pvalue > 1e-4
    table = np.zeros((k, k))
    np.add.at(table, (offs[0, :, 0], offs[1, :, 0]), 1)
    assert stats.chi2_contingency(table).pvalue > 1e-4, "state and next-state offsets are independent"


# ------------------------------------------------------------------------------------------------------------------------
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
                                               exp_avg_sq=o.exp_avg_sq, rng_counter=mem._rng_counter).items()}


LEARNER_CASES = {
    "c2": dict(),
    "c2-batch64-large-backward": dict(batch_size=64),
    "c3": dict(architecture="data-efficient", hidden_size=256, multi_step=20),
}


@pytest.mark.parametrize("case", list(LEARNER_CASES))
def test_learner_equals_unaugmented_twin_on_shifted_batch(case):
    """Three augmented learn() calls (two eager warm-ups, then the captured graph) against a twin without augmentation that
    samples the same batch, has its [s; s'] block replaced by the numpy shift at the offsets the augmented gather used, and
    runs the same update: losses, sum tree, parameters and both Adam moments bitwise after every update."""
    from rainbow_b200.memory import _SampleWorkspace
    kw = LEARNER_CASES[case]
    pad = 4
    aug, twin = _agent(augment_shift=pad, **kw), _agent(**kw)
    mem_kw = {k: v for k, v in kw.items() if k == "multi_step"}
    ma, mt = _memory(**mem_kw), _memory(**mem_kw)
    if case.startswith("c2-batch64"):
        assert aug.batch_size > 32   # k_head_bwd1's limit: the large-batch layer-1 kernels run
    assert aug._fused_path(aug.batch_size)
    B = aug.batch_size
    for step in range(3):
        aug.reset_noise()
        twin.reset_noise()
        aug.learn(ma)
        ws = _SampleWorkspace(B, mt.history, mt.device)
        mt.push_beta()
        mt.sample_into(ws)
        torch.cuda.synchronize()
        got = ma._last
        assert_bits_equal(cpu(ws.data_idx), cpu(got.data_idx), "sampled indices")
        sh = cpu(got.shifts)
        assert (sh != pad).any()
        both = np.concatenate([P.shift_ref(cpu(ws.states), sh[0], pad), P.shift_ref(cpu(ws.next_states), sh[1], pad)])
        ws.both_states.copy_(torch.from_numpy(both))
        assert_bits_equal(cpu(got.both_states), both, "the augmented learner's sampled states")
        loss = twin._update_from_batch(ws.as_tuple(), gate=ws.status,
                                       after_loss=lambda l: mt.update_priorities(ws.tree_idx, l, gate=ws.status))
        assert_bits_equal(cpu(aug.last_loss), cpu(loss), f"loss of update {step}")
        a, t = _snapshot(aug, ma), _snapshot(twin, mt)
        for k in a:
            assert_bits_equal(a[k], t[k], f"{k} after update {step}")
    assert set(aug._graphs) == {True}, "the third update ran as the captured graph"


def test_graph_replay_equals_eager():
    pad = 4
    ga, ea = _agent(augment_shift=pad), _agent(augment_shift=pad, cuda_graph=False)
    gm, em = _memory(), _memory()
    for step in range(7):
        for ag, mem in ((ga, gm), (ea, em)):
            ag.reset_noise()
            ag.learn(mem)
        assert_bits_equal(cpu(ga.last_loss), cpu(ea.last_loss), f"loss of update {step}")
        assert_bits_equal(cpu(gm._last.shifts), cpu(em._last.shifts), f"offsets of update {step}")
    assert ga._graphs and not ea._graphs
    g, e = _snapshot(ga, gm), _snapshot(ea, em)
    for k in g:
        assert_bits_equal(g[k], e[k], k)


_NODE = re.compile(r'label="\{KERNEL\s*\|\s*\{ID \| \d+ \(topoId: \d+\) \| ([^\\|<]+)')
_OWN = re.compile(r"(?<![A-Za-z_])k_[a-z0-9_]+")


def kernel_nodes(dot):
    """The function of every kernel node of a graph's DOT dump, in node order: the project's kernels by name (the mangled
    name's identifier, which ends before its first character outside [a-z0-9_]), library kernels by their mangled name."""
    out = []
    for func in _NODE.findall(html.unescape(dot)):
        own = _OWN.search(func)
        out.append(own.group(0) if own else func)
    return out


def update_graph(ag, mem, path, monkeypatch):
    """The kernels of the update graph learn() captures: two eager warm-up updates, then the capture (kept for its dump)."""
    orig = torch.cuda.CUDAGraph
    with monkeypatch.context() as m:
        m.setattr(torch.cuda, "CUDAGraph", functools.partial(orig, keep_graph=True))
        for _ in range(3):
            ag.reset_noise()
            ag.learn(mem)
    graph = ag._graphs[True][0]
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        graph.debug_dump(str(path))
    return kernel_nodes(open(path).read())


@pytest.mark.parametrize("batch", [32, 64])
def test_update_graph_swaps_only_the_gather(batch, tmp_path, monkeypatch):
    names = {}
    for tag, kw in (("default", dict()), ("off", dict(augment_shift=0)), ("on", dict(augment_shift=4))):
        names[tag] = update_graph(_agent(batch_size=batch, **kw), _memory(), tmp_path / f"{tag}.dot", monkeypatch)
    assert names["off"] == names["default"], "augment_shift = 0 leaves the update graph as it is"
    n = names["off"].count("k_gather")
    assert n >= 1 and "k_gather_shift" not in names["off"]
    assert names["on"].count("k_gather_shift") == n and "k_gather" not in names["on"]
    assert [("k_gather" if k == "k_gather_shift" else k) for k in names["on"]] == names["off"]
    assert len(names["off"]) >= 35 and sum(k.startswith("k_") for k in names["off"]) >= 20


def test_resume_equals_never_stopping(tmp_path):
    """5 augmented updates, save, fresh objects, load, 7 more == 12 uninterrupted updates, bitwise: the offsets depend only
    on the replay's seed and counter, which the checkpoint already holds."""
    from test_gpu_checkpoint import _agent as ck_agent
    from test_gpu_checkpoint import _assert_same, _before_update, _fresh_memory, _state, _update
    from test_gpu_checkpoint import _memory as ck_memory
    total, save_at = 12, 5
    ag, mem = ck_agent(augment_shift=4), ck_memory()
    losses = []
    for step in range(total):
        _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    run_a = _state(ag, mem, losses)

    ag, mem = ck_agent(augment_shift=4), ck_memory()
    losses = []
    for step in range(save_at):
        _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _before_update(ag, mem, save_at, True)
    ag.save_checkpoint(str(tmp_path / "ck"), mem)
    man = json.load(open(tmp_path / "ck" / "rank0" / "manifest.json"))
    assert man["hyper_parameters"]["augment_shift"] == 4
    ag, mem = ck_agent(seed=77, augment_shift=4), _fresh_memory()
    ag.load_checkpoint(str(tmp_path / "ck"), mem)
    for step in range(save_at, total):
        if step > save_at:
            _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _assert_same(run_a, _state(ag, mem, losses))

    plain = ck_agent()
    plain.save_checkpoint(str(tmp_path / "plain"))
    man = json.load(open(tmp_path / "plain" / "rank0" / "manifest.json"))
    assert "augment_shift" not in man["hyper_parameters"], "runs without augmentation write the manifest of before"


# ------------------------------------------------------------------------------------------------------------------------
def test_acting_and_evaluation_are_not_augmented():
    aug, plain = _agent(augment_shift=4, architecture="data-efficient", hidden_size=64), \
        _agent(architecture="data-efficient", hidden_size=64)
    val, _ = synthetic_ring(256, seed=4)
    states = val.iter_states(0, 8)
    for i in range(4):
        assert aug.act(states[i]) == plain.act(states[i])
    assert aug.evaluate_q_memory(val) == plain.evaluate_q_memory(val)
    a, b = aug.q_select(states), plain.q_select(states)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_refusals():
    from rainbow_b200 import RainbowB200Error
    for bad in (-1, 17):
        with pytest.raises(ValueError):
            _agent(augment_shift=bad, architecture="data-efficient", hidden_size=64)
    ag = _agent(augment_shift=4, architecture="data-efficient", hidden_size=64)
    mem, _ = synthetic_ring(1024, seed=5, rng="numpy")
    with pytest.raises(ValueError):
        ag.learn(mem)
    with pytest.raises(ValueError):
        mem.sample(8, shift_pad=4)
    philox, _ = synthetic_ring(1024, seed=5)
    with pytest.raises(ValueError):
        philox.sample(8, shift_pad=17)

    class Foreign:   # a reference-style host memory
        history = 4

        def sample(self, batch_size):
            raise AssertionError("not reached: the agent refuses first")

    with pytest.raises(RainbowB200Error):
        ag.learn(Foreign())
    assert int(ag.optimiser.step_count.item()) == 0, "a refused learn() does nothing"
