"""The noisy nets' device noise against the float64 reference of tests/noise_ref.py, per element, and the learner's draws
update by update.

* rb_noise_factors (k_noise_factors), device mode: the (n_in, n_out) of every net the agent builds (canonical /
  data-efficient x hidden 64 ... 2048 x 3 / 6 / 18 actions x 51 / 128 atoms), lengths 1 to 5 and around the 1024-thread
  CTA's pass of 4096 normals, counters 0, 1, 2^32 - 1, 2^32, 2^40 + 3 and seeds 0, 1, 2^32 + 5, 2^63 - 1, and 2^22 normals
  per stream once.  Every factor within noise_ref.factor_bound (TAU_X of the normal), no sign flip away from zero, the
  counter exactly one higher, guard elements past each output still NaN, a second launch bitwise equal, and a CUDA graph
  (k_noise_factors read from its nodes) replayed three times gives the eager draws at c, c + 1 and c + 2 bitwise.
  Injected mode: scale_noise(x) bitwise, counter untouched.
* rb_noisy_resample, device mode: bias_epsilon is rb_noise_factors' f_out at the same (seed, counter) bitwise, and
  weight_epsilon the fl32 outer product of those factors bitwise (so within the reference's bound too); k_bump_counter
  advances the counter once.  rb_noisy_outer: the fl32 outer product of given factors, bitwise.  Layer sets: both
  architectures' four layers, 1 to RB_MAX_NOISY_LAYERS layers (9 refused), in_f % 4 != 0 beside vector-path layers (Philox
  blocks straddle layers), a weight pointer one float off 16 B, in_f 3072 / 3073 with a ragged last CTA, in_f 57000 (the
  shared-memory staging limit) accepted and 57001 refused with nothing written.
* The learner, 9 learn() calls per case (two eager warm-ups, the capture, replays of both graph variants): fused head,
  library head and the data-efficient net with resets and ReDo, each with the online draw pending or flushed by an act().
  After every update both nets' factors are the reference's at (seed, counter before) within the bound, each counter
  one higher, the seeds noise_ref.agent_seeds; act / eval / evaluate_q launch at most the pending draw; a reset and a
  ReDo pass leave the counters alone; after load_checkpoint the next draws are the reference's at the restored counters;
  two ranks (torchrun, gloo on one GPU) draw from their own seeds.  The agent's captures collect garbage first and hold
  the collector off while they capture (a dead graph freed mid-capture invalidates it).
Observed largest |err| / bound go to $RB_PARITY_OBSERVED when that variable is set."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import noise_ref as N
from helpers import assert_bits_equal
from test_gpu_head_f64 import graph_kernels
from test_gpu_parity import DEV, FakeEnv, cpu, make_args, synthetic_ring

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN = float("nan")
GUARD = 5
COUNTERS = (0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 40 + 3)
SEEDS = (0, 1, 2 ** 32 + 5, 2 ** 63 - 1)
RB_ERR_RANGE = -34
ARCH_K1 = {"canonical": 3136, "data-efficient": 576}


@pytest.fixture(autouse=True)
def deterministic_cudnn():
    """The learner cases run deterministic cuDNN, like the other trajectory tests."""
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = old


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


def ptr(t):
    from rainbow_b200 import _lib
    return _lib.ptr(t)


def stream():
    return torch.cuda.current_stream().cuda_stream


def record(key, value):
    """Largest observed |err| / bound per output, merged into $RB_PARITY_OBSERVED."""
    path = os.environ.get("RB_PARITY_OBSERVED")
    if not path:
        return
    data = json.load(open(path)) if os.path.exists(path) else {}
    data.setdefault("noise_f64_tau_x", N.TAU_X)
    data[key] = max(float(value), data.get(key, 0.0))
    with open(path, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)


def counter(c):
    return torch.tensor([c], dtype=torch.int64, device=DEV)


def ctr_value(t):
    return int(t.item()) & (2 ** 64 - 1)


def check_draw(f_in, f_out, seed, c, tag):
    """Device factors (fp32, host) of draw c against the reference: (worst |err| / bound over both streams)."""
    x_in, r_in, x_out, r_out = N.draw(seed, c, f_in.size, f_out.size)
    worst = 0.0
    for name, f, x, r in (("f_in", f_in, x_in, r_in), ("f_out", f_out, x_out, r_out)):
        assert np.isfinite(f).all(), f"{tag}: {name} not finite"
        ratio, flips = N.factor_check(f, x, r)
        if ratio > 1.0 or flips:
            err = np.abs(f.astype(np.float64) - N.f64(x)) / N.factor_bound(x, r)
            i = int(err.argmax())
            pytest.fail(f"{tag}: {name}[{i}] = {f[i]!r}, reference f({x[i]!r}) = {N.f64(x[i])!r}: {ratio:.3g} x the bound, "
                        f"{flips} sign flips away from zero, {int((err > 1).sum())} of {f.size} over")
        worst = max(worst, ratio)
    return worst


# ---- rb_noise_factors ----------------------------------------------------------------------------------------------
def factors_launch(n_in, n_out, seed, ctr, x_in=None, x_out=None, bufs=None):
    """One rb_noise_factors launch into NaN-filled outputs with GUARD elements past each (or into `bufs`)."""
    if bufs is None:
        bufs = (torch.full((n_in + GUARD,), NAN, device=DEV), torch.full((n_out + GUARD,), NAN, device=DEV))
    rc = lib().rb_noise_factors(ptr(bufs[0]), n_in, ptr(bufs[1]), n_out, ptr(x_in), ptr(x_out), seed, ptr(ctr), stream())
    assert rc == 0, rc
    return bufs


def run_factors(n_in, n_out, seed, c, tag, tmp_path=None, graph=False):
    """The harness of one (n_in, n_out, seed, counter): eager draw vs the reference, guards, counter, second launch, and
    with graph=True three replays of a captured launch."""
    ctr = counter(c)
    fi, fo = factors_launch(n_in, n_out, seed, ctr)
    torch.cuda.synchronize()
    assert ctr_value(ctr) == (c + 1) & (2 ** 64 - 1), f"{tag}: counter advanced once"
    fi_h, fo_h = cpu(fi), cpu(fo)
    assert np.isnan(fi_h[n_in:]).all() and np.isnan(fo_h[n_out:]).all(), f"{tag}: guard elements written"
    worst = check_draw(fi_h[:n_in], fo_h[:n_out], seed, c, tag)
    ctr.fill_(c)
    fi2, fo2 = factors_launch(n_in, n_out, seed, ctr)
    torch.cuda.synchronize()
    assert_bits_equal(cpu(fi2), fi_h, f"{tag}: second launch f_in")
    assert_bits_equal(cpu(fo2), fo_h, f"{tag}: second launch f_out")
    if graph:
        eager = [(fi_h, fo_h)]
        for k in (1, 2):
            ctr.fill_(c + k)
            a, b = factors_launch(n_in, n_out, seed, ctr)
            eager.append((cpu(a), cpu(b)))
        ctr.fill_(c)
        gi, go = torch.full_like(fi, NAN), torch.full_like(fo, NAN)
        g, _, dot = graph_kernels(lambda: factors_launch(n_in, n_out, seed, ctr, bufs=(gi, go)), tmp_path / "factors.dot")
        assert "k_noise_factors" in dot, f"{tag}: the graph runs k_noise_factors"
        for k in range(3):            # graph_kernels replayed once already
            if k:
                g.replay()
                torch.cuda.synchronize()
            assert_bits_equal(cpu(gi), eager[k][0], f"{tag}: replay {k} f_in (draw c + {k})")
            assert_bits_equal(cpu(go), eager[k][1], f"{tag}: replay {k} f_out (draw c + {k})")
            assert ctr_value(ctr) == c + k + 1, f"{tag}: replay {k} counter"
    return worst


def _net_lengths(arch, hidden):
    K1 = ARCH_K1[arch]
    return [(2 * K1 + 2 * hidden, 2 * hidden + Z * (1 + A)) for A in (3, 6, 18) for Z in (51, 128)]


@pytest.mark.parametrize("hidden", [64, 256, 512, 1024, 2048])
@pytest.mark.parametrize("arch", ["canonical", "data-efficient"])
def test_factors_of_every_net(arch, hidden, tmp_path):
    worst = 0.0
    for i, (n_in, n_out) in enumerate(_net_lengths(arch, hidden)):
        seed, c = SEEDS[i % len(SEEDS)], COUNTERS[(i + hidden) % len(COUNTERS)]
        worst = max(worst, run_factors(n_in, n_out, seed, c, f"{arch}/{hidden} ({n_in}, {n_out}) seed {seed} ctr {c}",
                                       tmp_path, graph=i == 0))
    record("noise_factors / bound", worst)


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 4095, 4096, 4097, 3 * 4096 + 1])
def test_factors_lengths(n, tmp_path):
    worst = 0.0
    for j, m in enumerate((1, 5, 4097, n)):
        worst = max(worst, run_factors(n, m, SEEDS[j], COUNTERS[(n + j) % len(COUNTERS)], f"n_in {n} n_out {m}",
                                       tmp_path, graph=j == 3))
    record("noise_factors / bound", worst)


@pytest.mark.parametrize("seed", SEEDS)
def test_factors_counters_and_seeds(seed, tmp_path):
    worst = 0.0
    for c in COUNTERS:
        worst = max(worst, run_factors(4097, 13, seed, c, f"seed {seed} ctr {c}", tmp_path, graph=c == 2 ** 32 - 1))
    # the draws of distinct seeds and counters differ (the high words of both reach the key and the counter)
    ctr = counter(2 ** 32 + 7)
    a = cpu(factors_launch(64, 64, seed, ctr)[0])
    ctr.fill_(7)
    b = cpu(factors_launch(64, 64, seed, ctr)[0])
    c2 = counter(2 ** 32 + 7)
    d = cpu(factors_launch(64, 64, seed ^ (1 << 40), c2)[0])
    assert not np.array_equal(a, b) and not np.array_equal(a, d)
    record("noise_factors / bound", worst)


def test_factors_2_22_per_stream():
    """The statistical check of tests/test_noise_host.py on the device: 2^22 normals per stream, each within the bound."""
    n = 2 ** 22
    worst = run_factors(n, n, 2 ** 32 + 5, 2 ** 40 + 3, "2^22 per stream")
    record("noise_factors / bound", worst)


def test_factors_injected():
    rs = np.random.RandomState(3)
    for n_in, n_out in ((1, 1), (4097, 13), (6784, 1074)):
        x_in = rs.standard_normal(n_in).astype(np.float32)
        x_out = rs.standard_normal(n_out).astype(np.float32)
        edge = np.array([0.0, -0.0, 1e-45, -1e-45, 1e-38, 6.66, -6.66, 3e38], np.float32)
        x_in[:min(n_in, edge.size)] = edge[:min(n_in, edge.size)]
        ctr = counter(11)
        fi, fo = factors_launch(n_in, n_out, 123, ctr, torch.from_numpy(x_in).to(DEV), torch.from_numpy(x_out).to(DEV))
        torch.cuda.synchronize()
        assert ctr_value(ctr) == 11, "injected normals leave the counter alone"
        assert_bits_equal(cpu(fi)[:n_in], N.scale(x_in), "injected f_in")
        assert_bits_equal(cpu(fo)[:n_out], N.scale(x_out), "injected f_out")
        assert np.isnan(cpu(fi)[n_in:]).all() and np.isnan(cpu(fo)[n_out:]).all()


# ---- rb_noisy_resample / rb_noisy_outer -----------------------------------------------------------------------------
class Layers:
    """Weight and bias epsilon buffers of a layer set, NaN-filled with GUARD elements past each; `offset` floats in."""

    def __init__(self, shapes, offset=0):
        self.shapes = shapes
        self.w = [torch.full((offset + i * o + GUARD,), NAN, device=DEV) for i, o in shapes]
        self.b = [torch.full((o + GUARD,), NAN, device=DEV) for _, o in shapes]
        self.off = offset
        n = len(shapes)
        self.args = ((C.c_void_p * n)(*[t.data_ptr() + 4 * offset for t in self.w]),
                     (C.c_void_p * n)(*[t.data_ptr() for t in self.b]),
                     (C.c_int * n)(*[i for i, _ in shapes]), (C.c_int * n)(*[o for _, o in shapes]), n)

    def resample(self, seed, ctr):
        return lib().rb_noisy_resample(*self.args, None, None, seed, ptr(ctr), stream())

    def outer(self, f_in, f_out):
        return lib().rb_noisy_outer(*self.args, ptr(f_in), ptr(f_out), stream())

    def host(self):
        return [(cpu(w)[self.off:], cpu(b)) for w, b in zip(self.w, self.b)]

    def untouched(self):
        return all(np.isnan(w).all() and np.isnan(b).all() for w, b in self.host())

    def check(self, f_in, f_out, tag):
        """weight_epsilon == outer(f_out, f_in) and bias_epsilon == f_out per layer, bitwise; guards NaN."""
        oi = oo = 0
        for l, ((i, o), (w, b)) in enumerate(zip(self.shapes, self.host())):
            fi, fo = f_in[oi:oi + i], f_out[oo:oo + o]
            assert_bits_equal(b[:o], fo, f"{tag}: layer {l} bias_epsilon")
            assert_bits_equal(w[:i * o].reshape(o, i), N.outer(fo, fi), f"{tag}: layer {l} weight_epsilon")
            assert np.isnan(w[i * o:]).all() and np.isnan(b[o:]).all(), f"{tag}: layer {l} guards"
            oi, oo = oi + i, oo + o


def _arch_layers(arch, hidden, A, Z=51):
    K1 = ARCH_K1[arch]
    return [(K1, hidden), (K1, hidden), (hidden, Z), (hidden, A * Z)]


LAYER_SETS = {
    "canonical": _arch_layers("canonical", 512, 6),
    "data-efficient": _arch_layers("data-efficient", 256, 6),
    **{f"{n}-layers": [(8 + 12 * l + (l % 3), 3 + 5 * l) for l in range(n)] for n in range(1, 9)},
    "straddling": [(37, 19), (64, 5), (13, 70), (576, 64), (7, 3), (3, 9)],
    "in3072-in3073-ragged": [(3072, 8 * 5 + 3), (3073, 8 * 3 + 1), (5, 2)],
    "in57000": [(57000, 3), (4, 9)],
}


# every layer set aligned, and three of them with weight pointers one float off 16 B (the scalar path)
RESAMPLE_CASES = [(n, 0) for n in LAYER_SETS] + [(n, 1) for n in ("canonical", "straddling", "3-layers")]


@pytest.mark.parametrize("name,offset", RESAMPLE_CASES, ids=[f"{n}-offset{o}" for n, o in RESAMPLE_CASES])
def test_resample_equals_factors_and_outer(name, offset, tmp_path):
    shapes = LAYER_SETS[name]
    n_in, n_out = sum(i for i, _ in shapes), sum(o for _, o in shapes)
    worst = 0.0
    for k, (seed, c) in enumerate(((SEEDS[len(shapes) % 4], COUNTERS[len(shapes) % 5]), (2 ** 63 - 1, 2 ** 32 - 1))):
        tag = f"{name} offset {offset} seed {seed} ctr {c}"
        L = Layers(shapes, offset)
        ctr = counter(c)
        assert L.resample(seed, ctr) == 0
        torch.cuda.synchronize()
        assert ctr_value(ctr) == c + 1, f"{tag}: k_bump_counter advanced the counter once"
        fctr = counter(c)
        fi, fo = (cpu(t) for t in factors_launch(n_in, n_out, seed, fctr))
        fi, fo = fi[:n_in], fo[:n_out]
        L.check(fi, fo, tag)
        worst = max(worst, check_draw(fi, fo, seed, c, tag))
        if k == 0:
            # a second launch and a graph replay are bitwise equal; the graph holds the resample and the bump
            first = L.host()
            ctr.fill_(c)
            assert L.resample(seed, ctr) == 0
            torch.cuda.synchronize()
            for (w, b), (w0, b0) in zip(L.host(), first):
                assert_bits_equal(w, w0, f"{tag}: second launch")
                assert_bits_equal(b, b0, f"{tag}: second launch")
            ctr.fill_(c)
            for t in L.w + L.b:
                t.fill_(NAN)
            g, _, dot = graph_kernels(lambda: L.resample(seed, ctr), tmp_path / "resample.dot")
            assert "k_noisy_resample" in dot and "k_bump_counter" in dot, f"{tag}: graph nodes"
            assert ctr_value(ctr) == c + 1, f"{tag}: one replay, one bump"
            for (w, b), (w0, b0) in zip(L.host(), first):
                assert_bits_equal(w, w0, f"{tag}: graph replay")
                assert_bits_equal(b, b0, f"{tag}: graph replay")
    record("noisy_resample / bound", worst)


@pytest.mark.parametrize("name", ["canonical", "straddling", "8-layers", "in57000"])
def test_outer_of_given_factors(name):
    shapes = LAYER_SETS[name]
    n_in, n_out = sum(i for i, _ in shapes), sum(o for _, o in shapes)
    rs = np.random.RandomState(len(name))
    f_in = rs.standard_normal(n_in).astype(np.float32)
    f_out = rs.standard_normal(n_out).astype(np.float32)
    f_in[:4] = [0.0, -0.0, 1e-30, -3.0]
    for offset in (0, 1):
        L = Layers(shapes, offset)
        assert L.outer(torch.from_numpy(f_in).to(DEV), torch.from_numpy(f_out).to(DEV)) == 0
        torch.cuda.synchronize()
        L.check(f_in, f_out, f"{name} offset {offset}")


def test_resample_refusals():
    ctr = counter(5)
    nine = Layers([(8, 3)] * 9)
    assert nine.resample(1, ctr) == RB_ERR_RANGE, "RB_MAX_NOISY_LAYERS + 1 layers"
    big = Layers([(57001, 2), (4, 4)])
    assert big.resample(1, ctr) == RB_ERR_RANGE, "in_features above the shared-memory staging"
    f = torch.zeros(57005, device=DEV)
    assert big.outer(f, f) == RB_ERR_RANGE
    torch.cuda.synchronize()
    assert nine.untouched() and big.untouched() and ctr_value(ctr) == 5, "a refusal writes nothing"


# ---- the learner ----------------------------------------------------------------------------------------------------
LEARNER = {
    "fused": dict(),
    "library": dict(fused_head=False),
    "c3-reset-redo": dict(architecture="data-efficient", hidden_size=256, reset_interval=4, reset_shrink_encoder=0.5,
                          redo_interval=3),
}
CAP = 8192
UPDATES = 9


@pytest.fixture(scope="module")
def memory():
    mem, _ = synthetic_ring(CAP, seed=3)
    mem.seed = 99
    return mem


def _counters(ag):
    return ctr_value(ag.online_net._noise_counter), ctr_value(ag.target_net._noise_counter)


def _check_net(net, c, tag):
    return check_draw(cpu(net._f_in), cpu(net._f_out), net.noise_seed, c, tag)


def _learn_and_check(ag, mem, state, flush, tag):
    """reset_noise(); [act()]; learn(): each net drew once, at the counter it held before, from its own seed."""
    c_on, c_tg = _counters(ag)
    ag.reset_noise()
    if flush:
        ag.act(state)
        ag.act(state)
        torch.cuda.synchronize()
        assert _counters(ag) == (c_on + 1, c_tg), f"{tag}: act() launched the pending draw, once"
    ag.learn(mem)
    torch.cuda.synchronize()
    assert _counters(ag) == (c_on + 1, c_tg + 1), f"{tag}: counters {_counters(ag)} after ({c_on}, {c_tg})"
    return max(_check_net(ag.online_net, c_on, f"{tag}: online"), _check_net(ag.target_net, c_tg, f"{tag}: target"))


@pytest.mark.parametrize("noise", ["pending", "flushed"])
@pytest.mark.parametrize("case", list(LEARNER))
def test_learner_draws_update_by_update(case, noise, memory):
    from rainbow_b200.agent import Agent
    torch.manual_seed(5)
    ag = Agent(make_args(**LEARNER[case]), FakeEnv(6))
    assert (ag.online_net.noise_seed, ag.target_net.noise_seed) == N.agent_seeds(torch.initial_seed(), 0)
    assert ag._fused_path(ag.batch_size) == (case != "library")
    state = memory.iter_states(0, 1)[0]
    worst = 0.0
    for u in range(UPDATES):
        worst = max(worst, _learn_and_check(ag, memory, state, (noise == "flushed") != (u == 6), f"{case} update {u}"))
    assert set(ag._graphs) == {True, False}, "both captured variants ran"
    assert ag.reset_count == (2 if case == "c3-reset-redo" else 0) and ag.redo_count == (3 if case == "c3-reset-redo" else 0)
    # acting and evaluating draw nothing new
    before = _counters(ag)
    ag.act(state)
    ag.evaluate_q(state)
    ag.evaluate_q_batch(memory.iter_states(0, 3))
    ag.eval()
    ag.act(state)
    ag.evaluate_q(state)
    ag.train()
    torch.cuda.synchronize()
    assert _counters(ag) == before, "act / eval / evaluate_q launch no draw"
    # a reset and a ReDo pass leave both counters alone
    ag.reset_parameters(0.5, 0.2)
    ag.recycle_dormant()
    torch.cuda.synchronize()
    assert _counters(ag) == before, "reset / ReDo leave the noise counters alone"
    worst = max(worst, _learn_and_check(ag, memory, state, noise == "flushed", f"{case} after a reset"))
    record("learner noise / bound", worst)


def test_learner_draws_after_resume(memory, tmp_path):
    from rainbow_b200.agent import Agent
    torch.manual_seed(5)
    ag = Agent(make_args(), FakeEnv(6))
    state = memory.iter_states(0, 1)[0]
    for u in range(4):
        _learn_and_check(ag, memory, state, u == 2, f"before save, update {u}")
    ag.reset_noise()                                      # saved with the online draw pending
    ag.save_checkpoint(str(tmp_path / "ck"))
    seeds, ctrs = (ag.online_net.noise_seed, ag.target_net.noise_seed), _counters(ag)
    torch.manual_seed(11)
    fresh = Agent(make_args(), FakeEnv(6))
    assert (fresh.online_net.noise_seed, fresh.target_net.noise_seed) != seeds
    fresh.load_checkpoint(str(tmp_path / "ck"))
    assert (fresh.online_net.noise_seed, fresh.target_net.noise_seed) == seeds and _counters(fresh) == ctrs
    assert fresh.online_net._noise_pending
    fresh.learn(memory)                                   # the pending draw and the target's, at the restored counters
    torch.cuda.synchronize()
    assert _counters(fresh) == (ctrs[0] + 1, ctrs[1] + 1)
    worst = max(_check_net(fresh.online_net, ctrs[0], "resumed online"), _check_net(fresh.target_net, ctrs[1], "resumed target"))
    for u in range(3):
        worst = max(worst, _learn_and_check(fresh, memory, state, u == 1, f"after resume, update {u}"))
    record("learner noise / bound", worst)


class _Cycle:
    """A reference cycle: unreachable once dropped, freed only by the cyclic garbage collector."""

    def __init__(self):
        self.me = self


def test_captures_collect_dead_graphs_first(memory, monkeypatch):
    """The agent's update and act captures run the garbage collector before they begin and hold it off until they end: a
    dead cycle holding another CUDA graph (as a dropped Agent leaves behind) is freed before the capture, never by a
    collection an allocation inside it triggers -- destroying a graph while a stream captures invalidates the capture."""
    import gc
    import weakref
    from rainbow_b200.agent import Agent
    torch.manual_seed(5)
    ag = Agent(make_args(architecture="data-efficient", hidden_size=64), FakeEnv(6))
    seen = []

    def spy(name):
        orig = getattr(ag, name)

        def inner(*a, **kw):
            if torch.cuda.is_current_stream_capturing():
                seen.append((name, gc.isenabled(), dead() is None))
            return orig(*a, **kw)
        monkeypatch.setattr(ag, name, inner)
    spy("_sample_and_update")
    spy("q_select")
    cycle = _Cycle()
    cycle.graph = torch.cuda.CUDAGraph()
    x = torch.zeros(4, device=DEV)
    with torch.cuda.graph(cycle.graph):
        x.add_(1.0)
    gc.collect()                      # the cycle now sits in the oldest generation, which only a full collection frees
    dead = weakref.ref(cycle)
    del cycle
    state = memory.iter_states(0, 1)[0]
    for u in range(4):
        _learn_and_check(ag, memory, state, u == 3, f"update {u}")
    ag.act(state)                     # two act() calls warmed the act graph up: this one captures it
    assert sorted(n for n, _, _ in seen) == ["_sample_and_update", "_sample_and_update", "q_select"], seen
    assert all(not enabled for _, enabled, _ in seen), f"the collector ran free during a capture: {seen}"
    assert all(freed for _, _, freed in seen), f"a dead graph outlived the start of a capture: {seen}"
    assert gc.isenabled()


_DP_WORKER = r"""
import os, sys
import numpy as np
import torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
from rainbow_b200.dist import init_from_env
ngpu = torch.cuda.device_count()
backend = "nccl" if ngpu >= 2 else "gloo"          # one GPU: both ranks share it, gloo moves the CUDA tensors
if backend == "gloo":
    os.environ["LOCAL_RANK"] = "0"
rank, world, local = init_from_env(backend)
import noise_ref as N
from test_gpu_parity import FakeEnv, make_args, synthetic_ring
from rainbow_b200.agent import Agent
dev = torch.device("cuda", local)
torch.cuda.set_device(dev)
torch.manual_seed(7)                                # one torch seed on every rank, as a torchrun launch gives
args = make_args(device=dev, cuda_graph=False, architecture="data-efficient", hidden_size=64, batch_size=8,
                 peer_optimizer=False)
mem, _ = synthetic_ring(1024, seed=10, device=str(dev), args=dict(device=dev))
ag = Agent(args, FakeEnv(4))
on, tg = ag.online_net, ag.target_net
assert (on.noise_seed, tg.noise_seed) == N.agent_seeds(7, rank), (rank, on.noise_seed, tg.noise_seed)
for step in range(2):
    c = (int(on._noise_counter.item()), int(tg._noise_counter.item()))
    ag.reset_noise(); ag.learn(mem)
    torch.cuda.synchronize()
    assert (int(on._noise_counter.item()), int(tg._noise_counter.item())) == (c[0] + 1, c[1] + 1)
    for net, cc, what in ((on, c[0], "online"), (tg, c[1], "target")):
        f_in, f_out = net._f_in.cpu().numpy(), net._f_out.cpu().numpy()
        x_in, r_in, x_out, r_out = N.draw(net.noise_seed, cc, f_in.size, f_out.size)
        for f, x, r in ((f_in, x_in, r_in), (f_out, x_out, r_out)):
            ratio, flips = N.factor_check(f, x, r)
            assert ratio <= 1.0 and flips == 0, (rank, step, what, ratio, flips)
# the ranks' draws differ
mine = on._f_in[:256].double()
lo, hi = mine.clone(), mine.clone()
dist.all_reduce(lo, op=dist.ReduceOp.MIN); dist.all_reduce(hi, op=dist.ReduceOp.MAX)
assert not torch.equal(lo, hi), "the ranks drew the same noise"
dist.barrier()
dist.destroy_process_group()
print(f"rank{rank}ok backend={backend}", flush=True)
"""


def test_two_ranks_draw_from_their_own_seeds(tmp_path):
    script = tmp_path / "dp_noise.py"
    script.write_text(_DP_WORKER)
    port = 29500 + (os.getpid() + 97) % 190
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(script), ROOT]
    env = dict(os.environ, OMP_NUM_THREADS="1")
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-4000:]
    assert out.stdout.count("ok backend=") == 2, out.stdout
