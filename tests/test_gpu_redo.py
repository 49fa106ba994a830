"""Dormant-neuron statistics and ReDo recycling on the GPU: rb_neuron_scores against the float64 sums within its derived
bound, rb_redo_mask against the reference's mask on the kernel's own sums, rb_redo_recycle bitwise against the numpy
reference over both architectures' tables, and the learner with args.redo_interval: output preserved, schedule, graph
replay == eager, resume, two ranks."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import redo_ref as D
from helpers import assert_bits_equal
from test_gpu_augment import GUARD, update_graph
from test_gpu_parity import DEV, FakeEnv, cpu, make_args, synthetic_ring
from test_gpu_target_reset import C3, LEARNER_CASES, _assert_snapshots, _snapshot

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAP = 8192
TAUS = [0.0, 0.025, 0.1, 1.0]


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


def _agent(seed=5, **kw):
    from rainbow_b200.agent import Agent
    torch.manual_seed(seed)
    return Agent(make_args(**kw), FakeEnv(6))


def _memory(**args):
    mem, _ = synthetic_ring(CAP, seed=3, args=args)
    mem.seed = 99
    return mem


# ---- rb_neuron_scores ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1, 32, 512])
@pytest.mark.parametrize("C,HW", [(32, 400), (64, 81), (64, 49), (1024, 1)], ids=["conv1", "conv2", "conv3", "h"])
def test_scores_are_within_the_chunk_bound_of_float64(R, C, HW):
    rs = np.random.RandomState(R + C)
    act = np.maximum(rs.randn(R, C, HW).astype(np.float32) + 0.3, 0)
    act[:, 3] = 0.0
    a = torch.from_numpy(act).to(DEV)
    out = torch.full((C + 2 * GUARD,), -7.0, dtype=torch.float64, device=DEV)
    rc = lib().rb_neuron_scores(a.data_ptr(), R, C, HW, out.data_ptr() + 8 * GUARD, stream())
    assert rc == 0, lib().rb_last_error()
    got = cpu(out)
    assert (got[:GUARD] == -7.0).all() and (got[-GUARD:] == -7.0).all(), "guard elements"
    want = D.score_sums(act)
    # one fp32 chunk of 64 non-negative addends is within 63 * 2^-24 of its exact sum; the float64 tree adds 2^-53 per level
    assert (np.abs(got[GUARD:-GUARD] - want) <= D.SUM_REL_BOUND * want + 1e-12 * want).all()
    assert got[GUARD + 3] == 0.0
    again = torch.empty(C, dtype=torch.float64, device=DEV)
    lib().rb_neuron_scores(a.data_ptr(), R, C, HW, again.data_ptr(), stream())
    assert_bits_equal(cpu(again), got[GUARD:-GUARD], "a second launch sums in the same order")


# ---- rb_redo_mask ----------------------------------------------------------------------------------------------------------
def mask_launch(sums, layers, tau, k=0):
    from rainbow_b200 import _lib
    total = sums.numel()
    mask = torch.full((total + 2 * GUARD,), 9, dtype=torch.uint8, device=DEV)
    record = torch.full((_lib.REDO_RECORD_WORDS,), -1, dtype=torch.int64, device=DEV)
    arr = (_lib.RedoScored * len(layers))(*[_lib.RedoScored(*row) for row in layers])
    rc = lib().rb_redo_mask(sums.data_ptr(), arr, len(layers), tau, mask.data_ptr() + GUARD, record.data_ptr(), k, stream())
    assert rc == 0, lib().rb_last_error()
    m = cpu(mask)
    assert (m[:GUARD] == 9).all() and (m[-GUARD:] == 9).all(), "guard bytes"
    return m[GUARD:-GUARD], cpu(record)


@pytest.mark.parametrize("tau", TAUS)
def test_mask_and_counts_equal_the_reference_on_the_kernels_own_sums(tau):
    rs = np.random.RandomState(7)
    R = 32
    shapes = [(32, 400), (64, 81), (64, 49), (512, 1), (512, 1)]
    acts = [np.maximum(rs.randn(R, c, hw).astype(np.float32) * rs.rand(1, c, 1).astype(np.float32) - 0.2, 0)
            for c, hw in shapes]
    acts[1][:] = 0.0                      # a layer of all-zero activations: all dormant at every tau
    acts[2][:, 17] = 0.0                  # a single dead neuron
    acts[3][:] = 0.25                     # every score equals the mean: ties at the threshold when tau = 1
    offs = np.cumsum([0] + [c for c, _ in shapes])
    sums = torch.zeros(int(offs[-1]), dtype=torch.float64, device=DEV)
    for a, off, (c, hw) in zip(acts, offs, shapes):
        t = torch.from_numpy(a).to(DEV)
        assert lib().rb_neuron_scores(t.data_ptr(), R, c, hw, sums.data_ptr() + 8 * int(off), stream()) == 0
    layers = [(int(off), c, float(R * hw)) for off, (c, hw) in zip(offs, shapes)]
    got, record = mask_launch(sums, layers, tau, k=11)
    want, counts = D.mask_ref(cpu(sums), layers, tau)
    assert np.array_equal(got, want)
    assert record[:2].tolist() == [11, 5]
    assert record[2:12].reshape(5, 2).tolist() == [[c, n] for (c, _), n in zip(shapes, counts)]
    assert counts[1] == 64 and got[offs[2] + 17] == 1 and counts[2] >= 1
    assert counts[3] == (512 if tau == 1.0 else 0), "a score equal to the threshold is dormant (<=)"
    if tau == 0.0:
        assert counts[2] == int((D.score_sums(acts[2]) == 0).sum())


def test_mask_tie_exactly_at_a_fractional_threshold():
    sums = torch.tensor([0.5, 3.5, 2.0, 2.0, 0.0, 8.0], dtype=torch.float64, device=DEV)
    got, record = mask_launch(sums, [(0, 4, 1.0), (4, 2, 1.0)], 0.25)        # mean 2: the threshold is exactly 0.5
    assert got.tolist() == [1, 0, 0, 0, 1, 0] and record[2:6].tolist() == [4, 1, 2, 1]
    got, _ = mask_launch(sums, [(0, 4, 1.0), (4, 2, 1.0)], 0.125)
    assert got.tolist() == [0, 0, 0, 0, 1, 0]


# ---- rb_redo_recycle -------------------------------------------------------------------------------------------------------
def _host_net(arch):
    import argparse

    from rainbow_b200.agent import FusedClipAdam, redo_layers_c, redo_table
    from rainbow_b200.model import DQN
    torch.manual_seed(0)
    ns = argparse.Namespace(atoms=51, hidden_size=512 if arch == "canonical" else 256, architecture=arch, history_length=4,
                            noisy_std=0.1)
    net = DQN(ns, 6)
    opt = FusedClipAdam(net, lr=1e-4, eps=1e-4, max_norm=10.0)
    table = redo_table(net, opt.offsets)
    return opt, table, redo_layers_c(table)


def _patterns(table):
    total = table[-1]["mask_offset"] + table[-1]["neurons"]
    firsts = [r["mask_offset"] for r in table]
    lasts = [r["mask_offset"] + r["neurons"] - 1 for r in table]
    pats = {"none": [], "all": list(range(total)), "first": firsts, "last": lasts,
            "adjacent": [f + d for f in firsts for d in (3, 4)] + [lasts[0], firsts[1]],
            "one-layer-all": list(range(firsts[1], lasts[1] + 1))}
    out = {}
    for name, idx in pats.items():
        m = np.zeros(total, np.uint8)
        m[idx] = 1
        out[name] = m
    return out


@pytest.mark.parametrize("arch", ["canonical", "data-efficient"])
def test_recycle_equals_the_reference_bitwise(arch):
    opt, table, layers = _host_net(arch)
    n = opt.numel
    rs = np.random.RandomState(3)
    p0 = np.full(n + 2 * GUARD, 5.0, np.float32)
    p0[GUARD:-GUARD] = opt.flat_param.numpy()
    pad = np.ones(n, bool)
    for p, o in zip(opt.params, opt.offsets):
        pad[o:o + p.numel()] = False
    p0[GUARD:-GUARD][pad] = 3.0           # padding marked: it must come back as it was
    m0 = rs.randn(n + 2 * GUARD).astype(np.float32)
    v0 = rs.rand(n + 2 * GUARD).astype(np.float32)
    seed = 0x0123456789ABCDEF
    for k, (name, mask) in enumerate(_patterns(table).items()):
        bufs = [torch.from_numpy(x.copy()).to(DEV) for x in (p0, m0, v0)]
        dmask = torch.from_numpy(mask).to(DEV)
        rc = lib().rb_redo_recycle(*[b.data_ptr() + 4 * GUARD for b in bufs], n, layers, len(table), dmask.data_ptr(), seed, k,
                                   stream())
        assert rc == 0, lib().rb_last_error()
        wp, wm, wv, written = D.recycle_ref(p0[GUARD:-GUARD], m0[GUARD:-GUARD], v0[GUARD:-GUARD], table, mask, seed, k)
        for got, want, orig, what in zip(bufs, (wp, wm, wv), (p0, m0, v0), ("param", "exp_avg", "exp_avg_sq")):
            g = cpu(got)
            assert_bits_equal(g[GUARD:-GUARD], want, f"{what}, pattern {name}")
            assert_bits_equal(g[:GUARD], orig[:GUARD], f"{what} front guard")
            assert_bits_equal(g[-GUARD:], orig[-GUARD:], f"{what} back guard")
        assert not written[pad].any() and (wp[pad] == 3.0).all(), "padding is never written"
        assert written.any() == bool(mask.any())
        if name == "first":
            # the pass index is in the counter: the same mask with another index draws other values
            again = [torch.from_numpy(x.copy()).to(DEV) for x in (p0, m0, v0)]
            lib().rb_redo_recycle(*[b.data_ptr() + 4 * GUARD for b in again], n, layers, len(table), dmask.data_ptr(), seed,
                                  k + 1, stream())
            assert not np.array_equal(cpu(again[0]), cpu(bufs[0]))
            w1 = D.recycle_ref(p0[GUARD:-GUARD], m0[GUARD:-GUARD], v0[GUARD:-GUARD], table, mask, seed, k + 1)[0]
            assert_bits_equal(cpu(again[0])[GUARD:-GUARD], w1, "pass index + 1")
            # fresh incoming draws lie in [-b, b) and sigma equals its constant
            for row in table:
                for off, per, _, _, b, c in row["incoming"]:
                    x = wp[D.incoming_indices((off, per), 0)]
                    if row is table[0] or per == 1:
                        if b > 0:
                            assert (x >= -np.float32(b)).all() and (x < np.float32(b)).all()
                        else:
                            assert (x == np.float32(c)).all()


# ---- the learner -----------------------------------------------------------------------------------------------------------
def _kill(ag, conv_channels=(1, 5), hidden=(0, 7)):
    """Neurons dead by construction: conv channels with bias -1e6 (first and last conv layer), hidden neurons of both
    streams with zero incoming weights and bias, mu and sigma (dead under every noise draw)."""
    on = ag.online_net
    convs = on.conv_layers()
    with torch.no_grad():
        for m in (convs[0], convs[-1]):
            m.bias[list(conv_channels)] = -1e6
        for fc in (on.fc_h_v, on.fc_h_a):
            for t in (fc.weight_mu, fc.bias_mu, fc.weight_sigma, fc.bias_sigma):
                t[list(hidden)] = 0.0
    dead = {0: conv_channels, len(convs) - 1: conv_channels, len(convs): hidden, len(convs) + 1: hidden}
    return dead


def _everything_else(ag, mem):
    on, tg, o = ag.online_net, ag.target_net, ag.optimiser
    d = dict(step=o.step_count, target=ag.target_flat, tree=mem.transitions.tree, rng=mem._rng_counter,
             frames=mem.transitions.frames)
    if o.grouped:
        d["group_steps"] = o.group_steps
    for tag, net in (("online", on), ("target", tg)):
        d.update({f"{tag}.counter": net._noise_counter, f"{tag}.f_in": net._f_in, f"{tag}.f_out": net._f_out})
        d.update((f"{tag}.{n}", b) for n, b in net.named_buffers() if n.endswith("_epsilon"))
    torch.cuda.synchronize()
    return {k: cpu(v).copy() for k, v in d.items()}


def _z(ag, states, noisy):
    on = ag.online_net
    with torch.no_grad():
        x = on.features_nograd(states).contiguous()
        z, _, _ = on.head().forward(x, noisy=noisy)
        torch.cuda.synchronize()
        return cpu(z).copy()


@pytest.mark.parametrize("arch", ["canonical", "data-efficient"])
def test_a_pass_recycles_the_dead_and_preserves_the_output(arch):
    from rainbow_b200 import RainbowB200Error
    kw = dict() if arch == "canonical" else C3
    ag, mem = _agent(cuda_graph=False, **kw), _memory()
    with pytest.raises(RainbowB200Error, match="learn"):
        ag.recycle_dormant()
    assert ag.dormant_stats() == ([], None)
    for _ in range(2):
        ag.reset_noise()
        ag.learn(mem)
    on, o = ag.online_net, ag.optimiser
    on.flush_noise()
    dead = _kill(ag)
    ag.reset_noise()                                   # a draw is pending across the passes
    states = ag._redo_states
    z_train0, z_eval0 = _z_pending_safe(ag, states)
    before = _everything_else(ag, mem)
    bufs0 = [cpu(b).copy() for b in (o.flat_param, o.exp_avg, o.exp_avg_sq)]

    # scoring alone changes nothing, at any tau
    for tau in (0.0, 0.1, 1.0):
        ag.recycle_dormant(tau=tau, recycle=False)
        layers, k = ag.dormant_stats()
        rd = ag._redo
        R = states.shape[0]
        counts = [(r["mask_offset"], r["neurons"]) for r in rd["table"]]
        hw = [a.shape[2] * a.shape[3] for a in on.conv_forward_saving(states)[1:]] + [1, 1]
        want_mask, want_counts = D.mask_ref(cpu(rd["sums"]), [(off, n, float(R * p)) for (off, n), p in zip(counts, hw)], tau)
        assert k == 0 and [x[2] for x in layers] == want_counts and [x[1] for x in layers] == [n for _, n in counts]
        assert [x[0] for x in layers] == [r["name"] for r in rd["table"]]
        assert np.array_equal(cpu(rd["mask"]), want_mask)
    for b, b0, what in zip((o.flat_param, o.exp_avg, o.exp_avg_sq), bufs0, ("param", "exp_avg", "exp_avg_sq")):
        assert_bits_equal(cpu(b), b0, f"{what} after scoring alone")
    assert ag.redo_count == 0 and on._noise_pending
    # the scores are those of a float64 forward's activations, within the chunk bound (the conv layers' own rounding aside)
    acts = on.conv_forward_saving(states)
    for row, a in zip(rd["table"], acts[1:]):
        want = D.score_sums(cpu(a))
        got = cpu(rd["sums"])[row["mask_offset"]:row["mask_offset"] + row["neurons"]]
        assert (np.abs(got - want) <= 2 * D.SUM_REL_BOUND * want).all(), row["name"]

    # a pass over the constructed-dead neurons alone (the mask written here): z is unchanged under the noise factors too
    table = rd["table"]
    only = np.zeros(rd["mask"].numel(), np.uint8)
    for l, idx in dead.items():
        only[table[l]["mask_offset"] + np.array(idx)] = 1
    only_d = torch.from_numpy(only).to(DEV)
    rc = lib().rb_redo_recycle(o.flat_param.data_ptr(), o.exp_avg.data_ptr(), o.exp_avg_sq.data_ptr(), o.numel, rd["layers_c"],
                               len(table), only_d.data_ptr(), ag.reset_seed, 7, stream())
    assert rc == 0, lib().rb_last_error()
    torch.cuda.synchronize()
    wp, wm, wv, written = D.recycle_ref(*bufs0, table, only, ag.reset_seed, 7)
    assert_bits_equal(cpu(o.flat_param), wp, "parameters after the constructed pass")
    assert_bits_equal(cpu(o.exp_avg), wm, "exp_avg after the constructed pass")
    assert_bits_equal(cpu(o.exp_avg_sq), wv, "exp_avg_sq after the constructed pass")
    assert written.any() and (bufs0[1][written] != 0).any(), "the moments zeroed were not zero before"
    z_train1, z_eval1 = _z_pending_safe(ag, states)
    assert_bits_equal(z_train1, z_train0, "z in training mode, same noise factors")
    assert_bits_equal(z_eval1, z_eval0, "z in eval mode")
    convs = on.conv_layers()
    assert abs(convs[0].bias[1].item()) < 1.0, "the dead channel's bias was re-drawn"
    sigma = np.float32(on.fc_h_v.std_init / np.sqrt(on.fc_h_v.in_features))
    assert on.fc_h_v.weight_sigma[0, 0].item() == float(sigma) and on.fc_z_v.weight_sigma[0, 0].item() == 0.0

    # the learner's own pass at tau = 0: every exactly-dead neuron, the constructed ones (killed again) among them
    dead = _kill(ag)
    _, z_eval0 = _z_pending_safe(ag, states)
    bufs0 = [cpu(b).copy() for b in (o.flat_param, o.exp_avg, o.exp_avg_sq)]
    ag.recycle_dormant(tau=0.0)
    torch.cuda.synchronize()
    mask = cpu(rd["mask"])
    for l, idx in dead.items():
        assert mask[table[l]["mask_offset"] + np.array(idx)].all(), f"constructed-dead neurons of {table[l]['name']}"
    assert ag.redo_count == 1 and ag.dormant_stats()[1] == 0 and on._noise_pending
    wp, wm, wv, _ = D.recycle_ref(*bufs0, table, mask, ag.reset_seed, 0)
    assert_bits_equal(cpu(o.flat_param), wp, "parameters after the pass")
    assert_bits_equal(cpu(o.exp_avg), wm, "exp_avg after the pass")
    assert_bits_equal(cpu(o.exp_avg_sq), wv, "exp_avg_sq after the pass")
    after = _everything_else(ag, mem)
    for key in before:
        assert_bits_equal(after[key], before[key], f"{key} is untouched by a pass")
    assert_bits_equal(_z_pending_safe(ag, states)[1], z_eval0, "z in eval mode after the learner's pass")
    # the second pass draws with index 1
    _kill(ag, conv_channels=(2,), hidden=(3,))
    bufs1 = [cpu(b).copy() for b in (o.flat_param, o.exp_avg, o.exp_avg_sq)]
    ag.recycle_dormant(tau=0.0)
    torch.cuda.synchronize()
    assert ag.redo_count == 2 and ag.dormant_stats()[1] == 1
    want = D.recycle_ref(*bufs1, table, cpu(rd["mask"]), ag.reset_seed, 1)[0]
    assert_bits_equal(cpu(o.flat_param), want, "the second pass draws with index 1")
    with pytest.raises(ValueError):
        ag.recycle_dormant(tau=1.5)
    # the update that follows runs on the recycled net
    ag.learn(mem)
    torch.cuda.synchronize()
    assert np.isfinite(cpu(ag.last_loss)).all()


def _z_pending_safe(ag, states):
    """z in training mode (with the factors as they are, the pending draw kept pending) and in eval mode."""
    on = ag.online_net
    pending, on._noise_pending = on._noise_pending, False
    try:
        return _z(ag, states, True), _z(ag, states, False)
    finally:
        on._noise_pending = pending


def test_dormant_stats_does_not_perturb_the_following_update():
    a, b = _agent(cuda_graph=False, **C3), _agent(cuda_graph=False, **C3)
    ma, mb = _memory(), _memory()
    for step in range(4):
        for ag, mem in ((a, ma), (b, mb)):
            ag.reset_noise()
            ag.learn(mem)
        a.recycle_dormant(recycle=False)
        assert a.dormant_stats()[1] == 0
    _assert_snapshots(_snapshot(a, ma), _snapshot(b, mb), "with and without scoring passes")


def test_peer_optimiser_refuses_recycling_and_allows_scoring():
    from rainbow_b200 import RainbowB200Error
    ag, mem = _agent(cuda_graph=False, **C3), _memory()
    ag.reset_noise()
    ag.learn(mem)
    ag.optimiser.peer = object()          # what FusedClipAdam holds under the peer-memory optimiser
    p0 = cpu(ag.optimiser.flat_param).copy()
    with pytest.raises(RainbowB200Error, match="peer"):
        ag.recycle_dormant(tau=1.0)
    ag.recycle_dormant(tau=1.0, recycle=False)
    assert sum(x[2] for x in ag.dormant_stats()[0]) > 0
    assert_bits_equal(cpu(ag.optimiser.flat_param), p0, "a refused pass writes nothing")
    assert ag.redo_count == 0


def test_redo_interval_fires_after_every_nth_learn_after_the_reset(monkeypatch):
    ag, mem = _agent(redo_interval=3, redo_tau=0.5, reset_interval=6, architecture="data-efficient", hidden_size=64), _memory()
    calls = []
    orig_redo, orig_reset = ag.recycle_dormant, ag.reset_parameters
    monkeypatch.setattr(ag, "recycle_dormant", lambda *a, **k: (calls.append(("redo", ag._learn_calls)), orig_redo(*a, **k)))
    monkeypatch.setattr(ag, "reset_parameters", lambda *a: (calls.append(("reset", ag._learn_calls)), orig_reset(*a)))
    for _ in range(10):
        ag.reset_noise()
        ag.learn(mem)
    assert calls == [("redo", 3), ("reset", 6), ("redo", 6), ("redo", 9)]
    assert ag.redo_count == 3 and ag.dormant_stats()[1] == 2
    for bad in (dict(redo_interval=-1), dict(redo_interval=1.5), dict(redo_tau=1.5), dict(redo_tau=-0.1)):
        with pytest.raises(ValueError):
            _agent(architecture="data-efficient", hidden_size=64, **bad)


@pytest.mark.parametrize("case", list(LEARNER_CASES))
def test_graph_replays_after_a_pass_equal_eager_updates(case):
    kw, pending = LEARNER_CASES[case]
    kw = dict(kw, redo_interval=3, redo_tau=0.5)
    ga, ea = _agent(**kw), _agent(cuda_graph=False, **kw)
    gm, em = _memory(), _memory()
    for step in range(7):
        for ag, mem in ((ga, gm), (ea, em)):
            ag.reset_noise()
            if not pending:
                ag.online_net.flush_noise()
            ag.learn(mem)
        assert_bits_equal(cpu(ga.last_loss), cpu(ea.last_loss), f"loss of update {step}")
        _assert_snapshots(_snapshot(ga, gm), _snapshot(ea, em), f"after update {step}")
    assert ga._graphs and not ea._graphs and ga.redo_count == ea.redo_count == 2
    sa, sb = ga.dormant_stats(), ea.dormant_stats()
    assert sa == sb and sa[1] == 1 and sum(x[2] for x in sa[0]) > 0, "tau 0.5 finds dormant neurons: the passes wrote"


@pytest.mark.parametrize("batch", [32, 64])
def test_update_graph_is_the_graph_without_the_option(batch, tmp_path, monkeypatch):
    names = {}
    for tag, kw in (("default", dict()), ("zero", dict(redo_interval=0)), ("on", dict(redo_interval=1000, redo_tau=0.1))):
        names[tag] = update_graph(_agent(batch_size=batch, **kw), _memory(), tmp_path / f"{tag}.dot", monkeypatch)
    assert names["zero"] == names["default"] == names["on"], "recycling runs outside the update graph"
    assert not any("redo" in k or "neuron_scores" in k for k in names["on"])


def test_resume_equals_never_stopping(tmp_path):
    """Recycling every 4 updates at tau 0.5, data-efficient / 256: 5 updates, save, fresh objects under another torch seed,
    load, 7 more == 12 uninterrupted updates, bitwise.  Passes fall after updates 4 (before the save), 8 and 12."""
    from test_gpu_checkpoint import _agent as ck_agent
    from test_gpu_checkpoint import _assert_same, _before_update, _fresh_memory, _state, _update
    from test_gpu_checkpoint import _memory as ck_memory
    kw = dict(redo_interval=4, redo_tau=0.5, **C3)
    total, save_at = 12, 5
    ag, mem = ck_agent(**kw), ck_memory()
    losses = []
    for step in range(total):
        _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    run_a = _state(ag, mem, losses)
    assert ag.redo_count == 3 and sum(x[2] for x in ag.dormant_stats()[0]) > 0

    ag, mem = ck_agent(**kw), ck_memory()
    losses = []
    for step in range(save_at):
        _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _before_update(ag, mem, save_at, True)
    ag.save_checkpoint(str(tmp_path / "ck"), mem)
    man = json.load(open(tmp_path / "ck" / "rank0" / "manifest.json"))
    assert (man["hyper_parameters"]["redo_interval"], man["hyper_parameters"]["redo_tau"]) == (4, 0.5)
    assert man["learner"]["redo_count"] == 1
    ag, mem = ck_agent(seed=77, **kw), _fresh_memory()
    assert ag.redo_count == 0
    ag.load_checkpoint(str(tmp_path / "ck"), mem)
    assert ag.redo_count == 1
    for step in range(save_at, total):
        if step > save_at:
            _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _assert_same(run_a, _state(ag, mem, losses))
    assert ag.redo_count == 3


def test_manifest_without_redo_count_loads_as_zero(tmp_path):
    from rainbow_b200 import checkpoint as ckpt
    from test_gpu_checkpoint import _agent as ck_agent
    plain = ck_agent()
    plain.save_checkpoint(str(tmp_path / "plain"))
    path = tmp_path / "plain" / "rank0" / "manifest.json"
    man = json.load(open(path))
    assert "redo_count" not in man["learner"]
    assert "redo_interval" not in man["hyper_parameters"] and "redo_tau" not in man["hyper_parameters"]
    ag, mem = ck_agent(seed=9, redo_interval=4), _memory()
    ag.reset_noise()
    ag.learn(mem)
    ag.recycle_dormant(tau=1.0)
    assert ag.redo_count == 1
    ag.load_checkpoint(str(tmp_path / "plain"))
    assert ag.redo_count == 0
    man["learner"]["redo_count"] = -2
    man["digest"] = ckpt._digest(man)
    json.dump(man, open(path, "w"), indent=1, sort_keys=True)
    ag.redo_count = 5
    with pytest.raises(Exception, match="redo_count"):
        ag.load_checkpoint(str(tmp_path / "plain"))
    assert ag.redo_count == 5, "a refused load changes nothing"


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
def differs_somewhere(x, what):
    a = x.detach().to(dev, torch.float64)
    lo, hi = a.clone(), a.clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN); dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    assert not torch.equal(lo, hi), what
torch.manual_seed(7)
args = make_args(device=dev, cuda_graph=False, architecture="data-efficient", hidden_size=64, batch_size=8, redo_interval=3,
                 redo_tau=0.9)
mem, _ = synthetic_ring(1024, seed=10 + rank, device=str(dev), args=dict(device=dev))
mem.seed = 50 + rank                                # the ranks sample different batches of different rings
torch.manual_seed(100 + rank)
ag = Agent(args, FakeEnv(4))
for step in range(7):
    ag.reset_noise(); ag.learn(mem)
    torch.cuda.synchronize()
    if step == 1:
        # the ranks' own score sums differ (different batches): only the all-reduced sums give one mask
        before = ag.optimiser.flat_param.clone()
        world_size, ag.sync.enabled = ag.sync.world_size, False
        ag.sync.world_size = 1
        ag.recycle_dormant(recycle=False)
        differs_somewhere(ag._redo["sums"], "the ranks scored the same activations: the test cannot see a missing all-reduce")
        ag.sync.enabled, ag.sync.world_size = True, world_size
        assert torch.equal(before, ag.optimiser.flat_param)
    if step in (2, 5):
        same_everywhere(ag._redo["sums"], f"score sums differ after the pass of update {step}")
        same_everywhere(ag._redo["mask"], f"masks differ after the pass of update {step}")
        same_everywhere(ag._redo["record"], f"records differ after the pass of update {step}")
        assert sum(x[2] for x in ag.dormant_stats()[0]) > 0, "tau 0.9 finds dormant neurons"
    same_everywhere(ag.optimiser.flat_param, f"parameters diverged after update {step}")
    same_everywhere(ag.optimiser.exp_avg, f"exp_avg diverged after update {step}")
    same_everywhere(ag.optimiser.exp_avg_sq, f"exp_avg_sq diverged after update {step}")
assert ag.redo_count == 2
dist.barrier()
dist.destroy_process_group()
print(f"rank{rank}ok backend={backend}", flush=True)
"""


def test_two_ranks_form_one_mask_and_stay_identical(tmp_path):
    script = tmp_path / "dp_redo.py"
    script.write_text(_DP_WORKER)
    port = 29500 + os.getpid() % 190
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(script), ROOT]
    env = dict(os.environ, OMP_NUM_THREADS="1")
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-4000:]
    assert out.stdout.count("ok backend=") == 2, out.stdout
