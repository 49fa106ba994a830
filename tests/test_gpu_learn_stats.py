"""Per-update learner statistics: rb_learn_stats (k_learn_stats) and Agent.learn_stats().

The entry point runs on both logit layouts (the fused head's z = (z_value | z_advantage), the library path's q [B][A][Z])
with the loss and m of the distributional loss kernel on the inputs of tests/c51_ref.py (terminal rows, returns clamped to
Vmin and to Vmax, weights 0 and 1), and its record is compared against float64 values computed from the same fp32 inputs:
  loss_mean, objective, target_mean, edge_mass   float64 means of the fp32 inputs, scale = the mean of the magnitudes;
  q_mean                                         head_ref.expectation of the taken action's logits (c51_ref's scale);
each within TAU * scale (observed largest |err| / scale per field go to $RB_PARITY_OBSERVED when that variable is set).
loss_max, weight_min, grad_norm, clip_coef and applied must match exactly.  TAU is checked here
(test_tau_is_5x_above_the_fp32_model, CPU) against a numpy model of the kernel's arithmetic -- per-sample float32 terms,
float64 batch sums, one rounding -- on the same cases: TAU must be at least 5x its largest error / scale.

The learner tests check the records of eager and graph-replayed updates against the update's own tensors, bitwise equality
of graph replay and eager updates on the fused and library paths with and without a pending online-noise draw, that
recording leaves the update bitwise unchanged, and the record of a rejected batch."""
import numpy as np
import pytest
import torch

import c51_ref as C
import head_ref as R
from test_gpu_parity import DEV, FakeEnv, cpu, make_args, synthetic_ring

RB_ERR_INVAL, RB_ERR_RANGE = -22, -34
MAX_NORM = 10.0
TAU = 1e-6
MEANS = ("loss_mean", "objective", "q_mean", "target_mean", "edge_mass")
EXACT = ("loss_max", "weight_min", "grad_norm", "clip_coef", "applied")
REC_WORDS = 12          # 48-byte records
GUARD = 8               # records past the ring that must stay untouched

# (layout, B, A, Z, support, gate): B 1 / 32 / 512 on both layouts and 2048 through q, A 1 / 6 / 18, Z 2 / 51 / 128,
# gate NULL (None) / 1 / 0
CASES = [("z", 1, 6, 51, "pm10", None), ("z", 32, 6, 51, "pm10", 1), ("z", 512, 18, 51, "pm10", 0),
         ("z", 32, 1, 2, "pm10", None), ("z", 35, 18, 128, "m3to7", 1), ("z", 512, 6, 128, "pm100", None),
         ("q", 1, 1, 128, "pm10", 0), ("q", 32, 6, 51, "pm10", None), ("q", 512, 6, 2, "0to20", 1),
         ("q", 512, 18, 51, "m3to7", None), ("q", 2048, 6, 51, "pm10", 0), ("q", 35, 18, 128, "pm100", 1)]
NORMS = (37.5, 3.25)    # above and below MAX_NORM


def fields():
    from rainbow_b200 import _lib
    return np.dtype(_lib.LEARN_STATS_FIELDS)


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


def stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return None if t is None else t.data_ptr()


def case_inputs(case, device):
    layout, B, A, Z, sup, gate = case
    inp = C.make_inputs("dueling" if layout == "z" else "plain", B, A, Z, sup, seed=B * 1000 + A * 10 + Z)
    return C.to(inp, device)


def f64_loss_and_m(inp):
    """fp32 loss and m from the float64 reference (CPU: the inputs of the fp32 model; the GPU test uses the kernel's)."""
    ev, _ = C.expected_values(inp)
    m, _ = C.projection(inp, ev.argmax(1))
    m = m.float()
    (loss, _), _ = C.loss_grad(inp, m)
    return loss.float(), m


def reference(inp, loss, m):
    """{field: (float64 value, scale)} of the mean-type fields."""
    acts = inp["actions"]
    l, w, md, s = loss.double(), inp["weights"].double(), m.double(), inp["support"].double()
    q, L = C.logits(inp, "s")
    qa, La = C._row(q, acts), C._row(L, acts)
    lf = La + (qa - qa.max(-1, keepdim=True).values).abs()
    ev, evs = R.expectation(qa.unsqueeze(1), lf.unsqueeze(1), inp["support"])
    tv, tvs = (md * s).sum(1), (md.abs() * s.abs()).sum(1)
    edge, edges = md[:, 0] + md[:, -1], md[:, 0].abs() + md[:, -1].abs()
    return dict(loss_mean=(l.mean(), l.abs().mean()), objective=((w * l).mean(), (w * l).abs().mean()),
                q_mean=(ev.mean(), evs.mean()), target_mean=(tv.mean(), tvs.mean()), edge_mass=(edge.mean(), edges.mean()))


def exact(inp, loss, norm, gate):
    f = np.float32
    return dict(loss_max=f(loss.max().item()), weight_min=f(inp["weights"].min().item()), grad_norm=f(norm),
                clip_coef=min(f(MAX_NORM) / (f(norm) + f(1e-6)), f(1.0)), applied=f(0.0 if gate == 0 else 1.0))


def fp32_model(inp, loss, m):
    """The kernel's arithmetic in numpy: the dueling combination, the softmax expectation and sum m * support per sample
    in float32 (sequential sums, a coarser order than the kernel's warp butterflies), batch sums in float64, one rounding."""
    f, d = np.float32, np.float64
    B, A, Z = inp["B"], inp["A"], inp["Z"]
    acts, sup = inp["actions"].cpu().numpy(), inp["support"].cpu().numpy()
    rows = np.arange(B)
    if inp["entry"] == "plain":
        x = inp["q_on_s"].cpu().numpy()[rows, acts]
    else:
        zs = inp["z_on"][:B].cpu().numpy()
        za = zs[:, Z:].reshape(B, A, Z)
        mean = np.zeros((B, Z), f)
        for a in range(A):
            mean = mean + za[:, a]
        x = zs[:, :Z] + za[rows, acts] - mean / f(A)
    e = np.exp(x - x.max(1, keepdims=True))
    se, sn, tv = np.zeros(B, f), np.zeros(B, f), np.zeros(B, f)
    mm = m.cpu().numpy()
    for c in range(Z):
        se, sn, tv = se + e[:, c], sn + sup[c] * e[:, c], tv + mm[:, c] * sup[c]
    ev = sn / se
    l, w = loss.cpu().numpy().astype(d), inp["weights"].cpu().numpy().astype(d)
    return dict(loss_mean=f(l.mean()), objective=f((w * l).mean()), q_mean=f(ev.astype(d).mean()),
                target_mean=f(tv.astype(d).mean()), edge_mass=f((mm[:, 0] + mm[:, Z - 1]).astype(d).mean()))


def test_tau_is_5x_above_the_fp32_model():
    worst = {k: 0.0 for k in MEANS}
    for case in CASES:
        inp = case_inputs(case, "cpu")
        loss, m = f64_loss_and_m(inp)
        ref, got = reference(inp, loss, m), fp32_model(inp, loss, m)
        for k in MEANS:
            val, scale = ref[k]
            worst[k] = max(worst[k], abs(float(got[k]) - float(val)) / float(scale + C.FLOOR))
    assert max(worst.values()) > 0.0
    assert all(TAU >= 5 * v for v in worst.values()), worst


def test_record_layout_matches_the_header():
    import os
    import re
    from rainbow_b200 import _lib
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "rainbow_b200.h")).read()
    body = re.search(r"typedef struct rb_learn_stats_record \{(.*?)\} rb_learn_stats_record;", hdr, re.S).group(1)
    names = re.findall(r"\b(\w+)\s*[,;]", body)
    assert names == [n for n, _ in _lib.LEARN_STATS_FIELDS]
    assert fields().itemsize == _lib.LEARN_STATS_RECORD_BYTES == REC_WORDS * 4


def test_argument_codes_without_gpu():
    one = 8     # never dereferenced: validation fails first
    L = lib()
    # loss, weights, actions, m, support, z, q, B, A, Z, grad_norm, gate, max_norm, scratch, ring, capacity, counter, stream
    args = [one] * 5 + [one, None, 4, 6, 51, one, None, MAX_NORM, one, one, 4, one, None]
    for i in (0, 1, 2, 3, 4, 10, 13, 14, 16):            # null pointers
        a = list(args)
        a[i] = None
        assert L.rb_learn_stats(*a) == RB_ERR_INVAL, i
    a = list(args)
    a[6] = one
    assert L.rb_learn_stats(*a) == RB_ERR_INVAL          # both layouts
    a = list(args)
    a[5] = None
    assert L.rb_learn_stats(*a) == RB_ERR_INVAL          # neither
    a = list(args)
    a[9] = 129
    assert L.rb_learn_stats(*a) == RB_ERR_RANGE          # Z > RB_MAX_ATOMS
    a = list(args)
    a[15] = 0
    assert L.rb_learn_stats(*a) == RB_ERR_RANGE          # empty ring
    # the two halves on their own
    assert L.rb_learn_stats_batch(one, one, one, one, one, one, None, 4, 6, 51, None, None) == RB_ERR_INVAL
    assert L.rb_learn_stats_batch(one, one, one, one, one, one, one, 4, 6, 51, one, None) == RB_ERR_INVAL
    assert L.rb_learn_stats_write(one, one, None, MAX_NORM, one, 0, one, None) == RB_ERR_RANGE
    assert L.rb_learn_stats_write(None, one, None, MAX_NORM, one, 4, one, None) == RB_ERR_INVAL
    assert L.rb_learn_stats_scratch_elems() > 8


# ---- the entry point on the GPU ----------------------------------------------------------------------------------------
def new_ring(cap, start=0):
    """Ring of cap records + GUARD guard records, all bytes 0xff; counter [start, guard word]."""
    ring = torch.full(((cap + GUARD) * REC_WORDS,), -1, dtype=torch.int32, device=DEV)
    counter = torch.tensor([start, -7], dtype=torch.int64, device=DEV)
    return ring, counter


def records(ring):
    return cpu(ring).view(fields())


def new_scratch():
    return torch.zeros(lib().rb_learn_stats_scratch_elems(), dtype=torch.float64, device=DEV)


def launch(inp, layout, loss, m, norm_t, gate_t, ring, cap, counter, scratch):
    B, A, Z = inp["B"], inp["A"], inp["Z"]
    z = inp["z_on"] if layout == "z" else None
    q = inp["q_on_s"] if layout == "q" else None
    return lib().rb_learn_stats(loss.data_ptr(), inp["weights"].data_ptr(), inp["actions"].data_ptr(), m.data_ptr(),
                                inp["support"].data_ptr(), _ptr(z), _ptr(q), B, A, Z, norm_t.data_ptr(), _ptr(gate_t), MAX_NORM,
                                scratch.data_ptr(), ring.data_ptr(), cap, counter.data_ptr(), stream())


def kernel_inputs(case, k):
    from test_gpu_c51_f64 import run
    layout, B, A, Z, sup, gate = case
    inp = case_inputs(case, DEV)
    loss, _, m, _ = run(inp)               # the loss kernel's own outputs, with NaN guard rows past B
    norm = NORMS[k % 2]
    norm_t = torch.tensor([norm], dtype=torch.float32, device=DEV)
    gate_t = None if gate is None else torch.tensor([gate, 5, 5, 5], dtype=torch.int32, device=DEV)
    return inp, loss, m, norm, norm_t, gate_t


@pytest.mark.gpu
@pytest.mark.parametrize("k,case", list(enumerate(CASES)), ids=[f"{c[0]}-B{c[1]}-A{c[2]}-Z{c[3]}-{c[4]}-gate{c[5]}" for c in CASES])
def test_learn_stats_f64(k, case, tmp_path):
    from test_gpu_head_f64 import graph_kernels, record
    layout, B, A, Z, sup, gate = case
    inp, loss, m, norm, norm_t, gate_t = kernel_inputs(case, k)
    cap, start = 3, 5 + k
    ring, counter = new_ring(cap, start)
    scratch = new_scratch()
    assert launch(inp, layout, loss, m, norm_t, gate_t, ring, cap, counter, scratch) == 0, lib().rb_last_error()
    torch.cuda.synchronize()
    assert cpu(counter).tolist() == [start + 1, -7], "counter advanced by one, nothing written past it"
    rec = records(ring)
    slot = start % cap
    blank = np.full(1, -1, np.int32).repeat(REC_WORDS).view(fields())[0]
    for j in range(cap + GUARD):
        if j != slot:
            assert rec[j].tobytes() == blank.tobytes(), f"record {j} written (slot {slot})"
    r = rec[slot]
    assert int(r["update"]) == start

    ref = reference(inp, loss[:B], m[:B])
    for name in MEANS:
        val, scale = ref[name]
        err = abs(float(r[name]) - float(val))
        record(f"learn_stats.{name}", err / float(scale + C.FLOOR))
        assert err <= TAU * float(scale + C.FLOOR), f"{name}: {float(r[name])} vs {float(val)} (scale {float(scale)})"
    for name, want in exact(inp, loss[:B], norm, gate).items():
        assert np.float32(r[name]).tobytes() == np.float32(want).tobytes(), f"{name}: {r[name]} != {want}"
    if B >= 5:
        assert float(r["edge_mass"]) > 0.0, "clamped returns put mass on the end atoms"

    ring2, counter2 = new_ring(cap, start)
    scratch2 = new_scratch()
    _, _, dot = graph_kernels(lambda: launch(inp, layout, loss, m, norm_t, gate_t, ring2, cap, counter2, scratch2),
                              tmp_path / "s.dot")
    assert "k_learn_stats_batch" in dot and "k_learn_stats_record" in dot
    assert float(scratch2[-1]) == 0.0, "the completion ticket returns to zero"
    assert torch.equal(ring, ring2) and torch.equal(counter, counter2), "eager launch and graph replay differ"


@pytest.mark.gpu
def test_ring_wraps_and_counter_advances():
    case = ("z", 32, 6, 51, "pm10", 1)
    inp, loss, m, norm, norm_t, gate_t = kernel_inputs(case, 0)
    ring, counter, scratch = new_ring(4) + (new_scratch(),)
    for _ in range(10):
        assert launch(inp, "z", loss, m, norm_t, gate_t, ring, 4, counter, scratch) == 0
    torch.cuda.synchronize()
    assert cpu(counter).tolist() == [10, -7]
    rec = records(ring)
    assert rec["update"][:4].tolist() == [8, 9, 6, 7]
    assert (rec.view(np.int32).reshape(-1, REC_WORDS)[4:] == -1).all(), "guard records untouched"
    same = {tuple(np.float32(rec[j][f]).tobytes() for f in MEANS + EXACT) for j in range(4)}
    assert len(same) == 1, "same inputs, same record"


@pytest.mark.gpu
def test_refused_calls_write_nothing():
    case = ("q", 32, 6, 51, "pm10", None)
    inp, loss, m, norm, norm_t, gate_t = kernel_inputs(case, 0)
    ring, counter = new_ring(4, 2)
    L = lib()
    B, A, Z = 32, 6, 51
    scratch = new_scratch()
    base = [loss.data_ptr(), inp["weights"].data_ptr(), inp["actions"].data_ptr(), m.data_ptr(), inp["support"].data_ptr(),
            None, inp["q_on_s"].data_ptr(), B, A, Z, norm_t.data_ptr(), None, MAX_NORM, scratch.data_ptr(), ring.data_ptr(), 4,
            counter.data_ptr(), stream()]
    bad = [({0: None}, RB_ERR_INVAL), ({3: None}, RB_ERR_INVAL), ({10: None}, RB_ERR_INVAL), ({13: None}, RB_ERR_INVAL),
           ({14: None}, RB_ERR_INVAL), ({16: None}, RB_ERR_INVAL), ({5: inp["q_on_s"].data_ptr()}, RB_ERR_INVAL),
           ({6: None}, RB_ERR_INVAL), ({9: 129}, RB_ERR_RANGE), ({15: 0}, RB_ERR_RANGE), ({15: -3}, RB_ERR_RANGE)]
    for change, rc in bad:
        a = list(base)
        for i, v in change.items():
            a[i] = v
        assert L.rb_learn_stats(*a) == rc, (change, L.rb_last_error())
    torch.cuda.synchronize()
    assert (cpu(ring) == -1).all() and cpu(counter).tolist() == [2, -7], "a refused call writes nothing"
    assert float(scratch.abs().max()) == 0.0, "a refused call writes nothing"


# ---- the learner -------------------------------------------------------------------------------------------------------
def _agent(stats, graph=True, fused=True, B=32, **kw):
    from rainbow_b200.agent import Agent
    torch.manual_seed(5)
    args = make_args(cuda_graph=graph, batch_size=B, fused_head=fused, learn_stats=stats, **kw)
    return Agent(args, FakeEnv(6))


def _memory():
    mem, _ = synthetic_ring(8192, seed=3, args=dict())
    mem.seed = 99
    return mem


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [True, False], ids=["fused", "library"])
def test_agent_records_match_the_update_eager(fused):
    ag, mem = _agent(8, graph=False, fused=fused), _memory()
    assert ag._fused_path(32) == fused
    for k in range(4):
        ag.reset_noise()
        ag.learn(mem)
        rec = ag.learn_stats()
        assert rec["dropped"] == 0 and rec["update"].tolist() == [k]
        ws, loss = mem._last, ag.last_loss
        l, w = loss.double(), ws.weights.double()
        for name, (val, scale) in dict(loss_mean=(l.mean(), l.abs().mean()), objective=((w * l).mean(), (w * l).abs().mean())).items():
            assert abs(float(rec[name][0]) - float(val)) <= TAU * float(scale), name
        assert np.float32(rec["loss_max"][0]) == np.float32(loss.max().item())
        assert np.float32(rec["weight_min"][0]) == np.float32(ws.weights.min().item())
        assert _bits(rec["grad_norm"]).tobytes() == _bits(cpu(ag.optimiser.grad_norm)).tobytes()
        assert float(rec["applied"][0]) == float(cpu(ws.status)[0]) == 1.0
        assert int(ag.optimiser.step_count.item()) == k + 1
        # q(s, a), the target value and the end-atom mass against float64 from this update's own logits and m: the
        # learner must hand the kernel the s rows of the online logits and the m of this update
        last = ag._stats["last"]
        inp = dict(B=32, A=6, Z=51, actions=ws.actions, weights=ws.weights, support=ag.support)
        if fused:
            assert last["q"] is None and last["z"].shape == (64, 51 * 7)
            inp.update(entry="dueling", z_on=last["z"], z_tg=None)
        else:
            assert last["z"] is None and last["q"].shape == (32, 6, 51)
            inp.update(entry="plain", q_on_s=last["q"])
        ref = reference(inp, loss, last["m"])
        for name in ("q_mean", "target_mean", "edge_mass"):
            val, scale = ref[name]
            assert abs(float(rec[name][0]) - float(val)) <= TAU * float(scale + C.FLOOR), name


def _trajectory(graph, fused, pending, steps=7, stats=16):
    ag, mem = _agent(stats, graph=graph, fused=fused), _memory()
    losses = []
    for _ in range(steps):
        ag.reset_noise()
        if not pending:
            ag.online_net.flush_noise()       # as an act() between reset_noise() and learn() would
        ag.learn(mem)
        losses.append(ag.last_loss.clone())
    torch.cuda.synchronize()
    assert (ag._graph is not None) == graph
    if graph:
        assert set(ag._graphs) == {pending}
    opt = ag.optimiser
    state = (torch.stack(losses), mem.transitions.tree.clone(), opt.flat_param.clone(), opt.exp_avg.clone(),
             opt.exp_avg_sq.clone())
    return (ag.learn_stats() if stats else None), state


@pytest.mark.gpu
@pytest.mark.parametrize("fused,pending", [(True, True), (True, False), (False, False), (False, True)],
                         ids=["fused-pending", "fused-flushed", "library-flushed", "library-pending"])
def test_graph_records_equal_eager_bitwise(fused, pending):
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    try:
        re_, se = _trajectory(False, fused, pending)
        rg, sg = _trajectory(True, fused, pending)
    finally:
        torch.backends.cudnn.deterministic = old
    assert re_["update"].tolist() == rg["update"].tolist() == list(range(7)) and re_["dropped"] == rg["dropped"] == 0
    for name in MEANS + EXACT:
        assert _bits(re_[name]).tobytes() == _bits(rg[name]).tobytes(), f"{name}: graph replay and eager records differ"
    assert all(torch.equal(a, b) for a, b in zip(se, sg)), "the updates themselves differ"


@pytest.mark.gpu
def test_library_pending_graph_records_match_its_updates():
    """The library head with the online draw deferred into the update: each record of the graph run is held to that run's
    own per-step losses (test_graph_records_equal_eager_bitwise[library-pending] holds the run to an eager one)."""
    ag, mem = _agent(16, graph=True, fused=False), _memory()
    losses, norms = [], []
    for _ in range(7):
        ag.reset_noise()
        ag.learn(mem)
        losses.append(ag.last_loss.clone())
        norms.append(ag.optimiser.grad_norm.clone())
    assert set(ag._graphs) == {True}
    rec = ag.learn_stats()
    assert rec["update"].tolist() == list(range(7)) and (rec["applied"] == 1).all()
    for k, (loss, norm) in enumerate(zip(losses, norms)):
        l = loss.double()
        assert abs(float(rec["loss_mean"][k]) - float(l.mean())) <= TAU * float(l.abs().mean())
        assert np.float32(rec["loss_max"][k]) == np.float32(loss.max().item())
        assert _bits(rec["grad_norm"][k:k + 1]).tobytes() == _bits(cpu(norm)).tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [True, False], ids=["fused", "library"])
def test_recording_leaves_the_update_unchanged(fused):
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    try:
        _, off = _trajectory(True, fused, True, stats=0)
        rec, on = _trajectory(True, fused, True, stats=16)
    finally:
        torch.backends.cudnn.deterministic = old
    names = ("losses", "sum tree", "parameters", "exp_avg", "exp_avg_sq")
    for name, a, b in zip(names, off, on):
        assert torch.equal(a, b), f"{name} differ with the statistics on"
    assert len(rec["update"]) == 7


@pytest.mark.gpu
def test_ring_read_back_and_setting_changes():
    ag, mem = _agent(0), _memory()
    with pytest.raises(Exception, match="off"):
        ag.learn_stats()
    for _ in range(4):                       # warm-up, capture, replay without statistics
        ag.reset_noise()
        ag.learn(mem)
    ag.set_learn_stats(4)
    assert not ag._graphs, "a change drops the captured graphs"
    for _ in range(10):
        ag.reset_noise()
        ag.learn(mem)
    assert ag._graph is not None
    rec = ag.learn_stats()
    assert rec["update"].tolist() == [6, 7, 8, 9] and rec["dropped"] == 6
    for _ in range(2):
        ag.reset_noise()
        ag.learn(mem)
    rec = ag.learn_stats()
    assert rec["update"].tolist() == [10, 11] and rec["dropped"] == 0
    rec = ag.learn_stats()
    assert len(rec["update"]) == 0 and rec["dropped"] == 0
    ag.set_learn_stats(0)
    with pytest.raises(Exception, match="off"):
        ag.learn_stats()


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
def test_rejected_batch_record(use_graph):
    """The setup of test_rejected_batch_is_skipped_on_device: every draw fails, the batch is rejected, the step skipped."""
    from rainbow_b200.agent import Agent
    from rainbow_b200.memory import ReplayMemory
    torch.manual_seed(1)
    args = make_args(cuda_graph=use_graph, architecture="data-efficient", hidden_size=64, batch_size=8, learn_stats=8)
    mem = ReplayMemory(args, 256, max_attempts=3, seed=4)
    tr = mem.transitions
    tr.load_arrays(timestep=np.arange(256) % 50, action=np.zeros(256), reward=np.ones(256), nonterminal=np.ones(256), index=10,
                   full=True, t_episode=11)
    tr.frames.fill_(7)
    ag = Agent(args, FakeEnv(4))
    for _ in range(5):
        ag.reset_noise()
        ag.learn(mem)
    rec = ag.learn_stats()
    assert rec["update"].tolist() == list(range(5))
    assert (rec["applied"] == 0).all() and (rec["objective"] == 0).all() and (rec["weight_min"] == 0).all()
    assert np.isfinite(rec["grad_norm"]).all() and int(ag.optimiser.step_count.item()) == 0
    tr.update(np.arange(256) + tr.tree_start, np.full(256, 0.5, np.float32))
    ag.reset_noise()
    ag.learn(mem)
    rec = ag.learn_stats()
    assert rec["applied"].tolist() == [1.0] and int(ag.optimiser.step_count.item()) == 1 and float(rec["weight_min"][0]) > 0


@pytest.mark.gpu
def test_foreign_memory_records_applied():
    """A reference-style memory (host sampling, no gate): every record says applied."""
    ag, mem = _agent(4, graph=True), _memory()

    class Foreign:
        def sample(self, B):
            return mem.sample(B)

        def update_priorities(self, idxs, prios):
            pass

    f = Foreign()
    for _ in range(3):
        ag.reset_noise()
        ag.learn(f)
    rec = ag.learn_stats()
    assert rec["update"].tolist() == [0, 1, 2] and (rec["applied"] == 1).all()
    assert _bits(rec["grad_norm"][-1:]).tobytes() == _bits(cpu(ag.optimiser.grad_norm)).tobytes()


_DP_WORKER = r"""
import os, sys
import numpy as np, torch, torch.distributed as dist
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
def same_everywhere(x, what, expect=True):
    a = torch.as_tensor(np.asarray(x, np.float64)).to(dev)
    lo, hi = a.clone(), a.clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN); dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    assert torch.equal(lo, hi) == expect, what
torch.manual_seed(7)
mem, _ = synthetic_ring(1024, seed=10, device=str(dev), args=dict(device=dev))
variants = [False] + ([True] if ngpu >= 2 else [])   # the peer-memory optimiser needs a GPU per rank
for peer in variants:
    # gloo collectives cannot be captured into a CUDA graph; NCCL's can
    args = make_args(device=dev, cuda_graph=backend == "nccl", architecture="data-efficient", hidden_size=64, batch_size=8,
                     learn_stats=8, peer_optimizer=peer)
    ag = Agent(args, FakeEnv(4))
    assert ag.sync.enabled and ag.peer_optimizer == peer
    for k in range(5):
        ag.reset_noise(); ag.learn(mem)
        rec = ag.learn_stats()
        assert rec["update"].tolist() == [k] and rec["dropped"] == 0
        mine = ag.optimiser.grad_norm.cpu().numpy()
        assert rec["grad_norm"].view(np.uint32).tolist() == mine.view(np.uint32).tolist(), "grad_norm of this rank's optimiser"
        assert float(rec["applied"][0]) == 1.0
        same_everywhere(rec["grad_norm"], "every rank clips with the norm of the reduced gradient")
        same_everywhere(rec["loss_mean"], "each rank records its own batch", expect=False)
    print(f"rank{rank}ok peer={peer}", flush=True)
dist.barrier()
dist.destroy_process_group()
print(f"rank{rank}done backend={backend}", flush=True)
"""


@pytest.mark.gpu
def test_two_rank_records(tmp_path):
    """Data parallel (torchrun world 2; NCCL with two GPUs, else both ranks on this GPU with gloo): each rank keeps its own
    ring, records its own batch and the norm its own optimiser used -- on the NCCL path and, with a GPU per rank, on the
    peer-memory optimiser's path."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "dp_stats_worker.py"
    script.write_text(_DP_WORKER)
    port = 29500 + os.getpid() % 150
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(script), root]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=dict(os.environ, OMP_NUM_THREADS="1"))
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-4000:]
    assert out.stdout.count("done backend=") == 2 and out.stdout.count("ok peer=False") == 2, out.stdout
