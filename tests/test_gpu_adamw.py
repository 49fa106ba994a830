"""Clip + AdamW with Adam state per parameter group (rb_clip_adamw, rb_peer_adamw_gather, args.weight_decay,
args.reset_optimizer) on the GPU.

* rb_clip_adamw against tests/adamw_ref.py per element, one step at a time from the kernel's own state: P around the
  vector loop's grid-stride wrap and 6.9 M, misaligned buffers and P % 4 != 0 (the scalar path), 1 to 4 groups with
  boundaries one quad either side of the wrap, lambda 0 / 1e-2 / 0.1 at lr 1e-4 and 1e-3, group counts 0 / 9 / 10^6
  (distinct per group), gate NULL / 1 / 0 (0: nothing but the norm written, no count advanced).  The ticket is back at 0
  after every call; three graph replays equal three eager steps; every lambda = 0 with equal counts is rb_clip_adam's
  result bitwise, on the vector and the scalar path.
* rb_peer_adamw_gather through tests/peer_ref.World at W = 1, 2, 4, 8 (the learner's two segments, distinct lambda and
  counts): gred bitwise, parameters and moments within TAU, parameters bitwise equal on every rank, counts and epoch;
  lambda = 0 with equal counts is rb_peer_adam_gather bitwise.
* The learner: both options off leave the update graph as it is; lambda = 0 with reset_optimizer on is bitwise a plain
  agent before any reset; at lambda = 0.1 every eager update is adamw_ref's step from the update's own gradient and state;
  resets restart the groups they move; graph replays after a reset equal eager updates; a rejected batch moves nothing;
  resume; two ranks stay identical through decay and restarts, and a head-only and an encoder-only restart each zero
  exactly this rank's range of the restarted group (its shard of the group's segment under the peer optimiser) and set
  the right count to 0.
Deterministic cuDNN, like the other trajectory tests."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import adamw_ref as AW
import head_ref as R
import peer_ref as PR
from helpers import assert_bits_equal
from test_gpu_augment import update_graph
from test_gpu_clip_adam_f64 import VEC_WRAP
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


# ---- rb_clip_adamw ---------------------------------------------------------------------------------------------------------
def _groups_c(groups):
    from rainbow_b200 import _lib
    return (_lib.AdamGroup * len(groups))(*[_lib.AdamGroup(b, e, w) for b, e, w in groups])


def adamw_call(p, g, m, v, P, groups, step, gsteps, part, norm=None, gate=None, gs=1.0, max_norm=10.0, lr=1e-3,
               b1=0.9, b2=0.999, eps=1.5e-4):
    rc = lib().rb_clip_adamw(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), P, gs, max_norm, lr, b1, b2, eps,
                             _groups_c(groups), len(groups), step.data_ptr(), gsteps.data_ptr(), part.data_ptr(),
                             None if norm is None else norm.data_ptr(), None if gate is None else gate.data_ptr(), stream())
    assert rc == 0, lib().rb_last_error()


def _cuts(P, n):
    """n groups over [0, P): boundaries one quad either side of the wrap where it fits, else spread evenly."""
    want = [VEC_WRAP - 4, VEC_WRAP + 4, VEC_WRAP // 2][:n - 1]
    if not all(0 < c < P for c in want):
        want = [(P * (k + 1) // n) // 4 * 4 for k in range(n - 1)]
    return [0] + sorted(want) + [P]


# (P, offsets (p, g, m, v), n groups, lambdas, lr, counts, gate)
KCASES = [
    (4096, (0, 0, 0, 0), 2, (0.1, 0.0), 1e-3, (0, 9), None),
    (4099, (0, 0, 0, 0), 3, (0.01, 0.1, 0.0), 1e-4, (9, 0, 10 ** 6), None),
    (4096, (1, 0, 0, 0), 2, (0.0, 0.1), 1e-3, (10 ** 6, 9), 1),
    (4096, (0, 0, 3, 0), 4, (0.1, 0.01, 0.0, 0.1), 1e-3, (0, 9, 10 ** 6, 1), None),
    (VEC_WRAP + 8, (0, 0, 0, 0), 2, (0.1, 0.01), 1e-3, (9, 0), None),
    (VEC_WRAP + 8, (0, 0, 0, 0), 3, (0.01, 0.0, 0.1), 1e-4, (0, 10 ** 6, 9), 1),
    (VEC_WRAP + 8, (0, 0, 0, 0), 4, (0.1, 0.1, 0.01, 0.0), 1e-3, (10 ** 6, 9, 0, 3), None),
    (VEC_WRAP + 8, (0, 0, 0, 2), 4, (0.1, 0.0, 0.01, 0.1), 1e-3, (9, 0, 10 ** 6, 3), None),
    (VEC_WRAP + 3, (0, 0, 0, 0), 3, (0.1, 0.01, 0.0), 1e-4, (0, 9, 10 ** 6), None),
    (6_875_136, (0, 0, 0, 0), 2, (0.1, 0.01), 1e-4, (9, 10 ** 6), None),
    (6_875_136, (0, 0, 0, 0), 1, (0.1,), 1e-3, (9,), 1),
    (4096, (0, 0, 0, 0), 2, (0.1, 0.1), 1e-3, (9, 0), 0),
    (VEC_WRAP + 8, (0, 0, 0, 0), 4, (0.1, 0.1, 0.01, 0.0), 1e-3, (10 ** 6, 9, 0, 3), 0),
]


def _kid(c):
    P, offs, n, wds, lr, counts, gate = c
    return (f"P{P}" + ("-off" + "".join(map(str, offs)) if any(offs) else "") + f"-g{n}-wd{'_'.join(f'{w:g}' for w in wds)}"
            f"-lr{lr:g}-t{'_'.join(map(str, counts))}-gate{gate}")


def _kbuffers(P, offs):
    return [torch.full((P + 3,), float("nan"), device=DEV)[o:o + P] for o in offs]


@pytest.mark.parametrize("case", KCASES, ids=[_kid(c) for c in KCASES])
def test_clip_adamw_f64(case):
    P, offs, n, wds, lr, counts, gate_v = case
    gen = torch.Generator(device=DEV).manual_seed(KCASES.index(case))
    cuts = _cuts(P, n)
    groups = [(cuts[k], cuts[k + 1], wds[k]) for k in range(n)]
    p, g, m, v = _kbuffers(P, offs)
    p.copy_(torch.randn(P, device=DEV, generator=gen))
    p[::7] = 0.0
    m.copy_(torch.randn(P, device=DEV, generator=gen) * 0.03)
    v.copy_(torch.rand(P, device=DEV, generator=gen).add_(0.5) * 1e-2)
    for (b, e, _), t in zip(groups, counts):
        if t == 0:
            m[b:e].zero_(), v[b:e].zero_()
    step = torch.full((1,), 5, dtype=torch.int64, device=DEV)
    gsteps = torch.tensor(list(counts), dtype=torch.int64, device=DEV)
    part = torch.zeros(lib().rb_clip_adam_scratch_elems(), dtype=torch.float64, device=DEV)
    norm = torch.full((1,), float("nan"), device=DEV)
    gate = None if gate_v is None else torch.full((1,), gate_v, dtype=torch.int32, device=DEV)
    for it in range(2):
        g.copy_(torch.randn(P, device=DEV, generator=gen))
        max_norm = 0.5 * float(g.double().norm()) if it == 0 else 1e4
        p0, m0, v0 = p.clone(), m.clone(), v.clone()
        c0, s0 = gsteps.tolist(), int(step.item())
        adamw_call(p, g, m, v, P, groups, step, gsteps, part, norm, gate, max_norm=max_norm, lr=lr)
        torch.cuda.synchronize()
        assert int(part.view(torch.int64)[-1]) == 0, "the completion ticket is back to 0"
        ref = AW.clip_adamw(p0, g, m0, v0, groups, c0, 1.0, max_norm, lr, 0.9, 0.999, 1.5e-4)
        R.assert_within("norm", norm, torch.tensor([ref["norm"][0]], dtype=torch.float64, device=DEV),
                        torch.tensor([ref["norm"][1]], dtype=torch.float64, device=DEV), AW.TAU)
        if gate_v == 0:
            assert torch.equal(p, p0) and torch.equal(m, m0) and torch.equal(v, v0), "gate 0 left the state alone"
            assert gsteps.tolist() == c0 and int(step.item()) == s0, "gate 0 advances no count"
            continue
        assert gsteps.tolist() == [c + 1 for c in c0] and int(step.item()) == s0 + 1
        for name, got in (("m", m), ("v", v), ("p", p)):
            R.assert_within(name, got, *ref[name], AW.TAU)


@pytest.mark.parametrize("P,offs", [(VEC_WRAP + 8, (0, 0, 0, 0)), (4099, (0, 0, 0, 0)), (4096, (0, 1, 0, 0))],
                         ids=["vector", "scalar-P%4", "scalar-misaligned"])
def test_no_decay_equal_counts_is_clip_adam_bitwise(P, offs):
    gen = torch.Generator(device=DEV).manual_seed(P)
    init = [torch.randn(P, device=DEV, generator=gen) * s for s in (0.1, 1.0, 0.03)] + \
           [torch.rand(P, device=DEV, generator=gen) * 1e-2]
    groups = [(0, (P // 3) // 4 * 4, 0.0), ((P // 3) // 4 * 4, P, 0.0)]
    runs = []
    for grouped in (False, True):
        p, g, m, v = _kbuffers(P, offs)
        for dst, src in zip((p, g, m, v), init):
            dst.copy_(src)
        step = torch.full((1,), 9, dtype=torch.int64, device=DEV)
        gsteps = torch.tensor([9, 9], dtype=torch.int64, device=DEV)
        part = torch.zeros(lib().rb_clip_adam_scratch_elems(), dtype=torch.float64, device=DEV)
        norm = torch.zeros(1, device=DEV)
        for _ in range(3):
            if grouped:
                adamw_call(p, g, m, v, P, groups, step, gsteps, part, norm, max_norm=5.0)
            else:
                rc = lib().rb_clip_adam(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), P, 1.0, 5.0, 1e-3, 0.9, 0.999,
                                        1.5e-4, step.data_ptr(), part.data_ptr(), norm.data_ptr(), None, stream())
                assert rc == 0
        torch.cuda.synchronize()
        runs.append([cpu(t) for t in (p, m, v, norm, step)])
    for a, b in zip(*runs):
        assert_bits_equal(a, b, "rb_clip_adamw with lambda 0 and equal counts vs rb_clip_adam")


def test_clip_adamw_graph_replay_equals_eager():
    P = VEC_WRAP + 8
    gen = torch.Generator(device=DEV).manual_seed(3)
    state0 = [torch.randn(P, device=DEV, generator=gen) * 0.01, torch.zeros(P, device=DEV), torch.zeros(P, device=DEV)]
    g = torch.randn(P, device=DEV, generator=gen)
    groups = [(0, VEC_WRAP - 4, 0.1), (VEC_WRAP - 4, P, 0.01)]
    runs = []
    for graphed in (False, True):
        p, m, v = (t.clone() for t in state0)
        step = torch.zeros(1, dtype=torch.int64, device=DEV)
        gsteps = torch.tensor([0, 7], dtype=torch.int64, device=DEV)
        part = torch.zeros(lib().rb_clip_adam_scratch_elems(), dtype=torch.float64, device=DEV)
        norm = torch.zeros(1, device=DEV)
        fn = lambda: adamw_call(p, g, m, v, P, groups, step, gsteps, part, norm, max_norm=100.0)
        if graphed:
            graph = torch.cuda.CUDAGraph()
            torch.cuda.synchronize()
            with torch.cuda.graph(graph):
                fn()
            for _ in range(3):
                graph.replay()
        else:
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        assert int(step.item()) == 3 and gsteps.tolist() == [3, 10] and int(part.view(torch.int64)[-1]) == 0
        runs.append((p, m, v, norm))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


# ---- rb_peer_adamw_gather --------------------------------------------------------------------------------------------------
class WorldW(PR.World):
    """peer_ref.World whose Adam launch is rb_peer_adamw_gather with per-segment lambda and counts."""

    def __init__(self, world, segments, device, lib, wds, counts):
        super().__init__(world, segments, device, lib)
        import ctypes as C
        self.wd_c = (C.c_float * len(segments))(*wds)
        for rk in self.ranks:
            rk["seg_steps"] = torch.tensor(list(counts), dtype=torch.int64, device=device)

    def launch_adam(self, r, hyper, stream):
        from rainbow_b200 import _lib
        max_norm, lr, (b1, b2), eps = hyper
        _lib.check(self.lib.rb_peer_adamw_gather(
            self.peer_param, self.peer_flags, self.peer_norms, self.W, r, len(self.segments), self.seg_begin, self.seg_len,
            self.wd_c, self._p(r, "gred"), self._p(r, "exp_avg"), self._p(r, "exp_avg_sq"), max_norm, lr, b1, b2, eps,
            self._p(r, "step_count"), self._p(r, "seg_steps"), self._p(r, "epoch"), self._p(r, "scratch"),
            self._p(r, "grad_norm"), None, stream.cuda_stream))
        self._mark_launched(r, "adam")


def _init_world(w, seed):
    rs = np.random.RandomState(seed)
    p0 = torch.from_numpy((rs.standard_normal(w.P) * 0.5).astype(np.float32)).to(DEV)
    for rk in w.ranks:
        rk["param"][:w.P].copy_(p0)
    torch.cuda.synchronize()


def _load_grads(w, step):
    grads = []
    for r, rk in enumerate(w.ranks):
        gr = PR.step_grad(7, step, r, w.P, "normal")
        rk["grad"][:w.P].copy_(torch.from_numpy(gr).to(DEV))
        grads.append(gr)
    torch.cuda.synchronize()
    return grads


@pytest.mark.parametrize("W", [1, 2, 4, 8])
def test_peer_adamw_against_the_reference(W):
    segments = PR.learner_segments("data-efficient")
    wds, counts = (0.1, 0.01), (0, 9)
    hyper = (1.0, 1e-3, (0.9, 0.999), 1.5e-4)
    w = WorldW(W, segments, DEV, lib(), wds, counts)
    _init_world(w, W)
    side = torch.cuda.Stream()
    for t in range(1, 4):
        grads = _load_grads(w, t)
        before = w.snapshot()
        c0 = w.ranks[0]["seg_steps"].tolist()
        w.step(hyper, side)
        torch.cuda.synchronize()
        snaps = w.snapshot()
        ref_g = PR.reduced_grad(grads)
        for r, s in enumerate(snaps):
            assert s["step_count"] == t and s["epoch"] == t
            assert w.ranks[r]["seg_steps"].tolist() == [c + 1 for c in c0]
            assert not s["tickets"].any()
            assert_bits_equal(s["param"], snaps[0]["param"], f"rank {r} parameters vs rank 0")
            for fl, sh in PR.shard_slices(segments, W, r):
                assert_bits_equal(s["gred"][sh], ref_g[fl], f"rank {r} gred")
        tt = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
        g = tt(PR.flat_from_shards(snaps, segments, "gred"))
        m0, v0 = (tt(PR.flat_from_shards(before, segments, k)) for k in ("exp_avg", "exp_avg_sq"))
        # the flat buffer in address order: the learner's segments are [head, conv] -> groups [conv, head]
        order = sorted(range(len(segments)), key=lambda s: segments[s][0])
        groups = [(segments[s][0], segments[s][1], wds[s]) for s in order]
        ref = AW.clip_adamw(tt(before[0]["param"]), g, m0, v0, groups, [c0[s] for s in order], 1.0, hyper[0], hyper[1],
                            *hyper[2], hyper[3])
        for name, got in (("m", tt(PR.flat_from_shards(snaps, segments, "exp_avg"))),
                          ("v", tt(PR.flat_from_shards(snaps, segments, "exp_avg_sq"))), ("p", tt(snaps[0]["param"]))):
            R.assert_within(f"{name} after step {t}", got, *ref[name], AW.TAU)


@pytest.mark.parametrize("W", [1, 2])
def test_peer_adamw_without_decay_is_peer_adam_bitwise(W):
    segments = PR.learner_segments("data-efficient")
    hyper = (1.0, 1e-3, (0.9, 0.999), 1.5e-4)
    side = torch.cuda.Stream()
    out = []
    for grouped in (False, True):
        w = WorldW(W, segments, DEV, lib(), (0.0, 0.0), (0, 0)) if grouped else PR.World(W, segments, DEV, lib())
        _init_world(w, 11)
        for t in range(1, 4):
            _load_grads(w, t)
            w.step(hyper, side)
            torch.cuda.synchronize()
        out.append(w.snapshot())
    for a, b in zip(*out):
        for k in ("param", "exp_avg", "exp_avg_sq", "grad_norm"):
            assert_bits_equal(a[k], b[k], f"{k}: lambda 0 with equal counts vs rb_peer_adam_gather")


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
    d = dict(tree=mem.transitions.tree, flat_param=o.flat_param, exp_avg=o.exp_avg, exp_avg_sq=o.exp_avg_sq,
             step_count=o.step_count, target=ag.target_flat, rng_counter=mem._rng_counter)
    if o.grouped:
        d["group_steps"] = o.group_steps
    return {k: cpu(v).copy() for k, v in d.items()}


def _assert_snapshots(a, b, what, keys=None):
    for k in keys or a:
        assert_bits_equal(a[k], b[k], f"{k} {what}")


C3 = dict(architecture="data-efficient", hidden_size=256)


@pytest.mark.parametrize("batch", [32, 64])
def test_options_off_leave_the_update_graph(batch, tmp_path, monkeypatch):
    names = {}
    for tag, kw in (("default", dict()), ("off", dict(weight_decay=0.0, reset_optimizer=False)),
                    ("on", dict(weight_decay=0.1))):
        names[tag] = update_graph(_agent(batch_size=batch, **kw), _memory(), tmp_path / f"{tag}.dot", monkeypatch)
    assert names["off"] == names["default"]
    on = names["on"]
    assert on.count("k_clip_adamw") == 1 and "k_clip_adam" not in on and "k_clip_adamw" not in names["default"]
    assert [("k_clip_adam" if n == "k_clip_adamw" else n) for n in on] == names["default"]


def test_restart_option_without_decay_is_plain_adam_before_any_reset():
    """lambda = 0 and reset_optimizer on: 5 eager updates and 7 graph replays bitwise those of a plain agent."""
    for graph in (False, True):
        a, b = _agent(cuda_graph=graph), _agent(cuda_graph=graph, reset_optimizer=True)
        assert b.optimiser.grouped and not a.optimiser.grouped
        ma, mb = _memory(), _memory()
        for step in range(5 if not graph else 7):
            for ag, mem in ((a, ma), (b, mb)):
                ag.reset_noise()
                ag.learn(mem)
            assert_bits_equal(cpu(a.last_loss), cpu(b.last_loss), f"loss of update {step}")
        sa, sb = _snapshot(a, ma), _snapshot(b, mb)
        _assert_snapshots(sa, sb, "plain vs grouped", keys=list(sa))
        n = int(sb["step_count"][0])
        assert sb["group_steps"].tolist() == [n, n]


LEARNER_CASES = {
    "fused-pending": (dict(), True),
    "fused-flushed": (dict(), False),
    "batch64-large-backward": (dict(batch_size=64), True),
    "c3": (C3, True),
    "library-head": (dict(fused_head=False), False),
}


def _ref_groups(opt):
    return [(b, e, opt.weight_decay) for b, e in opt.groups]


@pytest.mark.parametrize("case", list(LEARNER_CASES))
def test_learner_update_is_adamw_ref(case):
    kw, pending = LEARNER_CASES[case]
    ag, mem = _agent(weight_decay=0.1, learning_rate=1e-3, cuda_graph=False, **kw), _memory()
    assert ag._fused_path(ag.batch_size) == (case != "library-head")
    o = ag.optimiser
    o.set_group_step_counts([4, 0])     # distinct counts: a group using the other's count would show
    for step in range(3):
        ag.reset_noise()
        if not pending:
            ag.online_net.flush_noise()
        torch.cuda.synchronize()
        p0, m0, v0 = o.flat_param.clone(), o.exp_avg.clone(), o.exp_avg_sq.clone()
        c0 = o.group_step_counts()
        ag.learn(mem)
        torch.cuda.synchronize()
        assert o.group_step_counts() == [c0[0] + 1, c0[1] + 1]
        ref = AW.clip_adamw(p0, o.flat_grad, m0, v0, _ref_groups(o), c0, 1.0, ag.norm_clip, o.lr, *o.betas, o.eps)
        for name, got in (("m", o.exp_avg), ("v", o.exp_avg_sq), ("p", o.flat_param)):
            R.assert_within(f"{name} of update {step}", got, *ref[name], AW.TAU)


@pytest.mark.parametrize("shrink", [(1.0, 0.0), (0.5, 0.0)], ids=["head-only", "both"])
def test_reset_restarts_the_groups_it_moves(shrink):
    from rainbow_b200.agent import ENCODER, HEAD
    ag, mem = _agent(weight_decay=0.1, reset_optimizer=True, cuda_graph=False, **C3), _memory()
    o = ag.optimiser
    for _ in range(3):
        ag.reset_noise()
        ag.learn(mem)
    before = _snapshot(ag, mem)
    ag.reset_parameters(*shrink)
    after = _snapshot(ag, mem)
    restarted = [g for g in (ENCODER, HEAD) if shrink[g] < 1.0]
    for g in (ENCODER, HEAD):
        b, e = o.groups[g]
        if g in restarted:
            assert not after["exp_avg"][b:e].any() and not after["exp_avg_sq"][b:e].any()
            assert after["group_steps"][g] == 0
        else:
            assert_bits_equal(after["exp_avg"][b:e], before["exp_avg"][b:e], "a group the reset keeps")
            assert_bits_equal(after["exp_avg_sq"][b:e], before["exp_avg_sq"][b:e], "a group the reset keeps")
            assert_bits_equal(after["flat_param"][b:e], before["flat_param"][b:e], "a group the reset keeps")
            assert after["group_steps"][g] == 3
    assert int(after["step_count"][0]) == 3
    # the next update is a first AdamW step (t = 1) for every restarted group
    ag.reset_noise()
    torch.cuda.synchronize()
    p0, m0, v0, c0 = o.flat_param.clone(), o.exp_avg.clone(), o.exp_avg_sq.clone(), o.group_step_counts()
    ag.learn(mem)
    torch.cuda.synchronize()
    ref = AW.clip_adamw(p0, o.flat_grad, m0, v0, _ref_groups(o), c0, 1.0, ag.norm_clip, o.lr, *o.betas, o.eps)
    for name, got in (("m", o.exp_avg), ("v", o.exp_avg_sq), ("p", o.flat_param)):
        R.assert_within(f"{name} after the restart", got, *ref[name], AW.TAU)
    assert o.group_step_counts() == [1 if g in restarted else 4 for g in (ENCODER, HEAD)]
    # a restart needs the group optimiser
    plain = _agent(cuda_graph=False, architecture="data-efficient", hidden_size=64)
    with pytest.raises(Exception, match="group optimiser"):
        plain.reset_parameters(restart_optimizer=True)
    plain.reset_parameters(restart_optimizer=False)


def test_graph_after_a_restart_equals_eager():
    kw = dict(weight_decay=0.1, reset_optimizer=True, target_tau=0.005)
    ga, ea = _agent(**kw), _agent(cuda_graph=False, **kw)
    gm, em = _memory(), _memory()
    for step in range(7):
        for ag, mem in ((ga, gm), (ea, em)):
            ag.reset_noise()
            ag.learn(mem)
            if step == 3:
                ag.reset_parameters(0.5, 0.0)
        assert_bits_equal(cpu(ga.last_loss), cpu(ea.last_loss), f"loss of update {step}")
        _assert_snapshots(_snapshot(ga, gm), _snapshot(ea, em), f"after update {step}")
    assert ga._graphs and ga.optimiser.group_step_counts() == [3, 3]


@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
def test_rejected_batch_moves_nothing(use_graph):
    from rainbow_b200.agent import Agent
    from rainbow_b200.memory import ReplayMemory
    torch.manual_seed(1)
    args = make_args(cuda_graph=use_graph, architecture="data-efficient", hidden_size=64, batch_size=8, weight_decay=0.1)
    mem = ReplayMemory(args, 256, max_attempts=3, seed=4)
    tr = mem.transitions
    tr.load_arrays(timestep=np.arange(256) % 50, action=np.zeros(256), reward=np.ones(256), nonterminal=np.ones(256), index=10,
                   full=True, t_episode=11)
    tr.frames.fill_(7)
    ag = Agent(args, FakeEnv(4))
    p0 = cpu(ag.optimiser.flat_param).copy()
    for _ in range(5):
        ag.reset_noise()
        ag.learn(mem)
    torch.cuda.synchronize()
    assert int(ag.optimiser.step_count.item()) == 0 and ag.optimiser.group_step_counts() == [0, 0]
    assert_bits_equal(cpu(ag.optimiser.flat_param), p0, "a rejected batch decays nothing")


def test_resume_equals_never_stopping(tmp_path):
    """lambda 0.1, tau 0.005, a reset every 4 updates with restart (encoder shrunk by 0.5), data-efficient / 256: 5 updates,
    save, fresh objects, load, 7 more == 12 uninterrupted updates, bitwise, group counts included."""
    from test_gpu_checkpoint import _agent as ck_agent
    from test_gpu_checkpoint import _assert_same, _before_update, _fresh_memory, _state, _update
    from test_gpu_checkpoint import _memory as ck_memory
    kw = dict(weight_decay=0.1, reset_optimizer=True, target_tau=0.005, reset_interval=4, reset_shrink_encoder=0.5, **C3)
    total, save_at = 12, 5

    def state(ag, mem, losses):
        s = _state(ag, mem, losses)
        s["group_steps"] = cpu(ag.optimiser.group_steps).copy()
        return s

    ag, mem = ck_agent(**kw), ck_memory()
    losses = []
    for step in range(total):
        _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    run_a = state(ag, mem, losses)
    assert ag.reset_count == 3 and ag.optimiser.group_step_counts() == [0, 0]

    ag, mem = ck_agent(**kw), ck_memory()
    losses = []
    for step in range(save_at):
        _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _before_update(ag, mem, save_at, True)
    ag.save_checkpoint(str(tmp_path / "ck"), mem)
    man = json.load(open(tmp_path / "ck" / "rank0" / "manifest.json"))
    assert (man["hyper_parameters"]["weight_decay"], man["hyper_parameters"]["reset_optimizer"]) == (0.1, True)
    assert man["learner"]["optimiser_group_steps"] == [1, 1] and man["learner"]["optimiser_step"] == 5
    ag, mem = ck_agent(seed=77, **kw), _fresh_memory()
    ag.load_checkpoint(str(tmp_path / "ck"), mem)
    assert ag.optimiser.group_step_counts() == [1, 1]
    for step in range(save_at, total):
        if step > save_at:
            _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _assert_same(run_a, state(ag, mem, losses))


def test_manifest_without_group_counts_loads_with_the_step(tmp_path):
    """A run without the group optimiser, resumed with it on: both counts start at optimiser_step."""
    from test_gpu_checkpoint import _agent as ck_agent
    from test_gpu_checkpoint import _memory as ck_memory
    plain, mem = ck_agent(architecture="data-efficient", hidden_size=64, cuda_graph=False), ck_memory()
    for _ in range(3):
        plain.reset_noise()
        plain.learn(mem)
    plain.save_checkpoint(str(tmp_path / "plain"))
    man = json.load(open(tmp_path / "plain" / "rank0" / "manifest.json"))
    assert "optimiser_group_steps" not in man["learner"] and "weight_decay" not in man["hyper_parameters"]
    ag = ck_agent(seed=9, architecture="data-efficient", hidden_size=64, weight_decay=0.1, reset_optimizer=True)
    ag.load_checkpoint(str(tmp_path / "plain"))
    assert ag.optimiser.group_step_counts() == [3, 3] and int(ag.optimiser.step_count.item()) == 3
    assert_bits_equal(cpu(ag.optimiser.flat_param), cpu(plain.optimiser.flat_param), "parameters")


# ---- two ranks -------------------------------------------------------------------------------------------------------------
_DP_WORKER = r"""
import os, sys
import torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
from rainbow_b200.dist import init_from_env
ngpu = torch.cuda.device_count()
backend = "nccl" if ngpu >= 2 else "gloo"
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
args = make_args(device=dev, cuda_graph=False, architecture="data-efficient", hidden_size=64, batch_size=8, weight_decay=0.1,
                 reset_optimizer=True, reset_interval=4, reset_shrink_encoder=0.5,
                 peer_optimizer="auto" if backend == "nccl" else False)
mem, _ = synthetic_ring(1024, seed=10, device=str(dev), args=dict(device=dev))
ag = Agent(args, FakeEnv(4))
o = ag.optimiser
assert o.grouped
def ranges():
    # [encoder, head] ranges of this rank's moment arrays, from the layout alone: the whole group (replicated), or this
    # rank's part of the group's segment (peer: segment 0 = head, then segment 1 = encoder, parts back to back)
    if o.peer is None:
        return slice(0, o.conv_end), slice(o.conv_end, o.numel)
    hp, ep = (o.numel - o.conv_end) // o.peer.world, o.conv_end // o.peer.world
    return slice(hp, hp + ep), slice(0, hp)
def update(what):
    ag.reset_noise(); ag.learn(mem)
    torch.cuda.synchronize()
    same_everywhere(o.flat_param, f"parameters diverged after {what}")
    same_everywhere(o.group_steps, f"group counts diverged after {what}")
for step in range(5):
    update(f"update {step}")
    if step == 3:   # the scheduled reset (shrink 0.5 on both groups) restarted both
        assert not o.exp_avg.any() and not o.exp_avg_sq.any() and o.group_step_counts() == [0, 0]
assert ag.reset_count == 1 and o.group_step_counts() == [1, 1], o.group_step_counts()
for alphas, restarted, counts in (((1.0, 0.0), 1, [1, 0]), ((0.5, 1.0), 0, [0, 1])):
    m0, v0 = o.exp_avg.clone(), o.exp_avg_sq.clone()
    ag.reset_parameters(*alphas)
    torch.cuda.synchronize()
    r = ranges()
    kept = r[1 - restarted]
    assert m0[r[restarted]].any(), "the restarted shard held moments"
    assert not o.exp_avg[r[restarted]].any() and not o.exp_avg_sq[r[restarted]].any(), f"{alphas}: shard not zeroed"
    assert torch.equal(o.exp_avg[kept], m0[kept]) and torch.equal(o.exp_avg_sq[kept], v0[kept]), f"{alphas}: other shard moved"
    assert o.group_step_counts() == counts, (alphas, o.group_step_counts())
    update(f"the restart {alphas}")
assert ag.reset_count == 3 and o.group_step_counts() == [1, 2], o.group_step_counts()
dist.barrier()
dist.destroy_process_group()
print(f"rank{rank}ok backend={backend} peer={ag.peer_optimizer}", flush=True)
"""


def test_two_ranks_stay_identical_through_decay_and_a_restart(tmp_path):
    script = tmp_path / "dp_adamw.py"
    script.write_text(_DP_WORKER)
    port = 29500 + (os.getpid() + 97) % 190
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(script), ROOT]
    env = dict(os.environ, OMP_NUM_THREADS="1")
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-4000:]
    assert out.stdout.count("ok backend=") == 2, out.stdout
