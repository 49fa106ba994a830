"""Whole learner updates against the float64 reference of tests/update_ref.py, update by update, over the pairwise table
of the agent's switches in tests/update_cases.py.

Each case runs 9 learn() calls -- two eager warm-ups, the capture, replays -- with the online noise draw deferred into
the update or flushed by an act() beforehand (update 6 takes the other way, so both captured variants run), and asserts
the kernels its captured graphs ran (gather variant, loss kernel, head backward).  After every update, each stage is fed
the learner's own fp32 state from before it, so errors do not compound:
  1. horizon and gather: (n, gamma) is horizon_ref.schedule at the updates since the last reset; the returns equal
     oracle.gather of the update's own indices within 1e-6, the nonterminals bitwise (annealed: fl32(nt fl32(gamma^n)));
  2. loss within 1e-5 of float64 (or update_ref.TAU_LOSS of its scale, for large quantile losses); the double-DQN arg-max
     is taken on the learner's own online s' rows, and where astar_ok accepts two actions the learner matches one of the
     references; the sum-tree leaves are fl32(sqrt(loss)) bitwise, the last write of a duplicate winning;
  3. gradients: per element |g - g64| <= TAU_G scale (update_ref) for the head, every conv bias and conv layer 0's weight
     where rb_conv_wgrad computes it; cuDNN's conv weight gradients normwise (conv_ref.wgrad_normwise, TAU_LIB);
  4. optimiser: flat_param, exp_avg, exp_avg_sq within adam_ref / adamw_ref TAU of the step on the learner's own
     flat_grad; step and group counts one more than before;
  5. target: bitwise ema_ref(target before, parameters after the step) under tau; unchanged under a hard copy except at
     the copy, where it is the online net bitwise;
  6. reset and ReDo where they fire: parameters bitwise reset_ref / recycle_ref of the state they were applied to with the
     draw index the agent used; restarted groups have zero moments and counts, the others keep both; ReDo's mask is mask_ref of the scores of
     that update's own sampled states;
  7. learn statistics: the record's loss mean and objective within 1e-5 of float64, its gradient norm the optimiser's.
Deterministic cuDNN, like the other trajectory tests."""
import functools
import time
import warnings

import numpy as np
import pytest
import torch

import conv_ref as CR
import horizon_ref as HR
import oracle
import redo_ref as RD
import reset_ref as RR
import update_ref as U
from helpers import assert_bits_equal
from test_gpu_augment import kernel_nodes
from test_gpu_parity import FakeEnv, cpu, make_args, synthetic_ring
from update_cases import ANNEAL, CASES, HARD_COPY_AT, agent_kwargs, case_id

pytestmark = pytest.mark.gpu

CAP = 8192
UPDATES = 9
TOL_LOSS = 1e-5


@pytest.fixture(autouse=True)
def deterministic_cudnn():
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = old


@functools.lru_cache(maxsize=None)
def _memory_and_oracle(annealed):
    """The replay (fresh per case: priorities change) and an oracle ring holding the same records (built once)."""
    mem = _memory(annealed)
    tr = mem.transitions
    ref = oracle.OracleTree(CAP)
    for name in ("frames", "timestep", "action", "reward", "nonterminal"):
        getattr(ref, name)[:] = cpu(getattr(tr, name)).reshape(getattr(ref, name).shape)
    return ref


def _memory(annealed):
    mem, _ = synthetic_ring(CAP, seed=3, args=ANNEAL if annealed else {})
    mem.seed = 99
    return mem


def _state(ag):
    o = ag.optimiser
    s = dict(flat_param=o.flat_param.clone(), exp_avg=o.exp_avg.clone(), exp_avg_sq=o.exp_avg_sq.clone(),
             step_count=int(o.step_count.item()), target=ag.target_flat.clone(), reset_count=ag.reset_count,
             redo_count=ag.redo_count)
    s["group_steps"] = o.group_step_counts() if o.grouped else None
    return s


def _sides(ag, ws, p_before):
    """(conv masks, hidden masks) of the learner's own fp32 forward of the update's online rows [s; s'], with the
    parameters it updated from: conv_ref.conv_masks, and the hidden layer's sides as the update's own fused head forward
    left them in its h buffer (its split-K sums need not repeat bitwise), or from the library's NoisyLinear layers."""
    on, opt = ag.online_net, ag.optimiser
    H, rows = on.hidden_size, ws.both_states.shape[0]
    if ag._fused_path(ws.B):
        h = on.head()._scratch[rows]["h"].clone()
    masks = CR.conv_masks(ag, ws, p_before)
    if not ag._fused_path(ws.B):
        p_after = opt.flat_param.clone()
        opt.flat_param.copy_(p_before)
        with torch.no_grad():
            x = torch.cat([on.features(ws.states), on.features(ws.next_states)])
            h = torch.cat([on.fc_h_v(x), on.fc_h_a(x)], 1)
        opt.flat_param.copy_(p_after)
    return masks, [(h[:, :H] > 0).double(), (h[:, H:] > 0).double()]


def _own_ns_rows(ag, ws):
    """(q, L) of the online s' rows the loss kernel's arg-max read: the update's own fused head output, left in the
    head's z buffer for its row count ([s; s'] on the fused path, s' alone on the library path)."""
    on = ag.online_net
    M, K = ag.augment_copies
    fused = ag._fused_path(ws.B)
    z = on.head()._scratch[(M + K) * ws.B if fused else K * ws.B]["z"]
    return U.own_ns_logits((z[M * ws.B:] if fused else z).double(), on.action_space, on.atoms)


def _per_element(ag, ref):
    """Largest |g - g64| / scale over the head's gradients, for the reference `ref` (or an alternative)."""
    on, opt = ag.online_net, ag.optimiser
    worst = 0.0
    for (n, p), off in zip(on.named_parameters(), opt.offsets):
        if n.startswith("convs"):
            continue
        g = opt.flat_grad[off:off + p.numel()].view_as(p)
        worst = max(worst, U.ratio(g, ref["grads"][n], ref["scales"][n]))
    return worst


def _nearest(ag, ref):
    """Where the stage tests' arg-max rule accepts several actions for a row, the reference the learner's gradient is
    nearest; its scales are the base reference's."""
    best = min([ref] + ref["alternatives"], key=lambda r: _per_element(ag, dict(r, scales=ref["scales"])))
    return dict(ref, **{k: best[k] for k in ("loss", "lscale", "grads", "convs", "astar", "target")})


def _check_gradients(ag, ws, ref, fused, tag, seen):
    on, opt = ag.online_net, ag.optimiser
    convs = U.conv_names(on)
    own0 = fused and on._own_wgrad_ok(on.conv_layers()[0], ws.states)     # layer 0 through rb_conv_wgrad
    for (n, p), off in zip(on.named_parameters(), opt.offsets):
        g = opt.flat_grad[off:off + p.numel()].view_as(p)
        li = next((i for i, (wn, _) in enumerate(convs) if n == wn), None)
        if li is not None and not (li == 0 and own0):
            m = on.conv_layers()[li]
            gp, a = ref["convs"][li]
            wn = CR.wgrad_normwise(gp, a, m.kernel_size[0], m.stride[0])
            r = U.ratio(g, ref["grads"][n], wn)
            assert r <= CR.TAU_LIB, f"{tag}: cuDNN weight gradient {n} {r:.3g} of its normwise scale"
            key = "conv weight (cuDNN, normwise)"
        else:
            r = U.ratio(g, ref["grads"][n], ref["scales"][n])
            if r > U.TAU_G:
                e = torch.nan_to_num((g.double() - ref["grads"][n]).abs() / ref["scales"][n], nan=0.0).reshape(-1)
                i = int(e.argmax())
                pytest.fail(f"{tag}: gradient of {n} {r:.3g} x its scale at element {i} of {p.shape} (got "
                            f"{float(g.reshape(-1)[i]):.9g}, float64 {float(ref['grads'][n].reshape(-1)[i]):.9g}, scale "
                            f"{float(ref['scales'][n].reshape(-1)[i]):.3g}; {int((e > U.TAU_G).sum())} elements over)")
            key = n.split(".")[-1] if not n.startswith("convs") else ("conv bias" if n.endswith("bias") else "conv layer 0 weight")
        seen[key] = max(seen.get(key, 0.0), r)


def _check_optimiser(ag, before, mid, tag):
    opt = ag.optimiser
    ref = U.optimiser_ref(opt, before, opt.flat_grad)
    tau = U.AR.TAU
    for k in ("p", "m", "v"):
        got = mid[{"p": "flat_param", "m": "exp_avg", "v": "exp_avg_sq"}[k]]
        r = U.ratio(got, *ref[k])
        assert r <= tau, f"{tag}: {k} after the optimiser step {r:.3g} x its scale"
    assert mid["step_count"] == before["step_count"] + 1, tag
    if opt.grouped:
        assert mid["group_steps"] == [c + 1 for c in before["group_steps"]], tag


def _check_reset(ag, mid, after, tag):
    from rainbow_b200.agent import ENCODER, HEAD, reset_table
    alphas = ag.reset_shrink
    segs = [(off, n, b, c, alphas[g]) for off, n, b, c, g in reset_table(ag.online_net, ag.optimiser.offsets)]
    want, _ = RR.reset_ref(cpu(mid["flat_param"]), segs, ag.reset_seed, mid["reset_count"])
    assert_bits_equal(cpu(after["flat_param"]), want, f"{tag}: reset parameters")
    assert after["reset_count"] == mid["reset_count"] + 1
    opt = ag.optimiser
    for g in (ENCODER, HEAD):
        rng = slice(*opt.groups[g]) if opt.grouped else slice(0, opt.numel)
        if ag.reset_optimizer and alphas[g] < 1.0:
            assert not after["exp_avg"][rng].any() and not after["exp_avg_sq"][rng].any(), f"{tag}: group {g} restarted"
            assert after["group_steps"][g] == 0, f"{tag}: group {g} count restarted"
        else:
            if opt.grouped:
                assert after["group_steps"][g] == mid["group_steps"][g], f"{tag}: group {g} count kept"
            assert torch.equal(after["exp_avg"][rng], mid["exp_avg"][rng]), f"{tag}: group {g} moments kept"
            assert torch.equal(after["exp_avg_sq"][rng], mid["exp_avg_sq"][rng]), f"{tag}: group {g} moments kept"


def _check_redo(ag, ws, mid, after, tag):
    """ReDo on the update's own rows of s: scores from the learner's fp32 forward of ws.states with the parameters of the
    pass, mask_ref away from the threshold, and recycle_ref of the kernel's mask bitwise."""
    on, opt = ag.online_net, ag.optimiser
    assert ag._redo_states.data_ptr() == ws.states.data_ptr(), f"{tag}: ReDo scores the update's own states"
    rd = ag._redo
    table = rd["table"]
    p_after = opt.flat_param.clone()
    opt.flat_param.copy_(mid["flat_param"])
    with torch.no_grad():
        acts = on.conv_forward_saving(ws.states)
        feats = acts[-1].reshape(ws.states.shape[0], -1)
        h = torch.cat([torch.relu(torch.nn.functional.linear(feats, m.weight_mu, m.bias_mu)) for m in (on.fc_h_v, on.fc_h_a)], 1)
    opt.flat_param.copy_(p_after)
    sums = np.concatenate([RD.score_sums(cpu(a)) for a in acts[1:]] + [RD.score_sums(cpu(h))])
    R = ws.states.shape[0]
    layers = [(row["mask_offset"], row["neurons"], R * (a.shape[2] * a.shape[3] if a is not None else 1))
              for row, a in zip(table, acts[1:] + [None, None])]
    want, _ = RD.mask_ref(sums, layers, ag.redo_tau)
    got = cpu(rd["mask"])
    clear = np.ones(got.size, bool)
    for off, n, count in layers:
        s = RD.normalised_scores(sums[off:off + n], count)
        clear[off:off + n] = np.abs(s - np.float32(ag.redo_tau)) > 4 * RD.SUM_REL_BOUND * (1 + np.abs(s))
    assert_bits_equal(got[clear], want[clear], f"{tag}: ReDo mask")
    p, m, v, _ = RD.recycle_ref(cpu(mid["flat_param"]), cpu(mid["exp_avg"]), cpu(mid["exp_avg_sq"]), table, got,
                                ag.reset_seed, mid["redo_count"])
    assert_bits_equal(cpu(after["flat_param"]), p, f"{tag}: recycled parameters")
    assert_bits_equal(cpu(after["exp_avg"]), m, f"{tag}: recycled exp_avg")
    assert_bits_equal(cpu(after["exp_avg_sq"]), v, f"{tag}: recycled exp_avg_sq")
    assert after["redo_count"] == mid["redo_count"] + 1


def _check_gather(ag, ws, ref_ring, horizon, tag):
    n, g = horizon
    gp = np.array([g ** k for k in range(n)], np.float32)
    _, _, ret, _, nt = oracle.gather(ref_ring, cpu(ws.data_idx), ag.history, n, gp)
    np.testing.assert_allclose(cpu(ws.returns), ret, rtol=0, atol=1e-6, err_msg=f"{tag}: returns")
    want = nt.reshape(-1) if ag._horizon is None else (nt.reshape(-1) * np.float32(g ** n)).astype(np.float32)
    assert_bits_equal(cpu(ws.nonterminals).reshape(-1), want, f"{tag}: nonterminals")


def _kernels(graph, path):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        graph.debug_dump(str(path))
    return kernel_nodes(open(path).read())


def _expected_kernels(c, ag):
    gather = {"none": "k_gather", "shift": "k_gather_shift", "intensity": "k_gather_aug", "drq": "k_gather_aug"}[c["aug"]]
    if c["horizon"] == "annealed":
        gather += "_hz"
    fused = c["head"] == "fused"
    M = ag.augment_copies[0]
    if c["dist"] == "quantile":
        loss = "k_qr_dueling" if fused else "k_qr"
    else:
        loss = ("k_c51_dueling_avg" if M > 1 else "k_c51_dueling") if fused else "k_c51"
    bwd = (["k_head_bwd1"] if M * c["batch"] <= 32 else ["k_head_bwd1_wgrad", "k_head_bwd1_dx"]) if fused else []
    return gather, loss, bwd


@pytest.mark.parametrize("c", CASES, ids=[case_id(c) for c in CASES])
def test_update_trajectory_against_float64(c, tmp_path, monkeypatch):
    from rainbow_b200.agent import Agent
    t0 = time.time()
    torch.manual_seed(5)
    ag = Agent(make_args(**agent_kwargs(c)), FakeEnv(6))
    annealed = c["horizon"] == "annealed"
    ref_ring = _memory_and_oracle(annealed)
    mem = _memory(annealed)
    on, tg, opt = ag.online_net, ag.target_net, ag.optimiser
    fused = c["head"] == "fused"
    M, K = ag.augment_copies
    assert ag._fused_path(ag.batch_size) == fused and mem.priority_exponent == 0.5
    act_state = mem.iter_states(0, 1)[0]

    # the state each reset / ReDo pass was applied to
    mids = []
    for name in ("reset_parameters", "recycle_dormant"):
        orig = getattr(ag, name)

        def wrapped(*a, _orig=orig, _name=name, **kw):
            mids.append((_name, _state(ag)))
            return _orig(*a, **kw)
        monkeypatch.setattr(ag, name, wrapped)
    monkeypatch.setattr(torch.cuda, "CUDAGraph", functools.partial(torch.cuda.CUDAGraph, keep_graph=True))

    since_reset, seen, ties = 0, {}, 0
    for u in range(UPDATES):
        tag = f"{case_id(c)} update {u}"
        ag.reset_noise()
        if (c["noise"] == "flushed") != (u == 6):
            ag.act(act_state)
        if c["target"] == "hard" and u == HARD_COPY_AT:
            ag.update_target_net()
            assert torch.equal(ag.target_flat, opt.flat_param), f"{tag}: the hard copy is the online net"
        torch.cuda.synchronize()
        horizon = ag.horizon()
        if annealed:
            want = HR.schedule(since_reset, ANNEAL["anneal_steps"], ANNEAL["multi_step_start"], ANNEAL["multi_step"],
                               ANNEAL["discount_start"], ANNEAL["discount"])
            assert horizon[0] == want[0] and horizon[1] == pytest.approx(want[1], rel=1e-12, abs=0), tag
        else:
            assert horizon == (3, 0.99), tag
        before = _state(ag)
        before_named = {n: p.detach().clone() for n, p in on.named_parameters()}
        target_named = {n: p.detach().clone() for n, p in tg.named_parameters()}
        mids.clear()
        ag.learn(mem)
        torch.cuda.synchronize()
        after = _state(ag)
        ws = mem._last
        B = ws.B
        assert int(ws.status[0].item()) == 1, f"{tag}: batch accepted"
        # the state right after the optimiser step: before the first reset / ReDo pass of this learn(), if any
        mid = mids[0][1] if mids else after

        _check_gather(ag, ws, ref_ring, horizon, tag)
        sides = _sides(ag, ws, before["flat_param"])
        f_on, f_tg = on.noise_factors(), tg.noise_factors()
        batch = dict(actions=ws.actions, returns=ws.returns, nonterminals=ws.nonterminals, weights=ws.weights,
                     gamma_n=ag._gamma_n())
        if ag.quantile:
            batch.update(kappa=ag.quantile_kappa)
        else:
            batch.update(support=ag.support, vmin=ag.Vmin, vmax=ag.Vmax, dz=ag.delta_z)
        ref = U.update_ref(on, before_named, f_on, ws.both_states, sides, tg, target_named, f_tg, ws.next_states, batch,
                           ag.distribution, M, K, own_ns=_own_ns_rows(ag, ws))
        ties += len(ref["ties"])
        ref = _nearest(ag, ref)
        err = (ag.last_loss.double() - ref["loss"]).abs()
        seen["loss (abs)"] = max(seen.get("loss (abs)", 0.0), float(err.max()))
        seen["loss / scale"] = max(seen.get("loss / scale", 0.0), float((err / ref["lscale"]).max()))
        # the north-star 1e-5, or for a large (quantile) loss TAU_LOSS of its scale: fp32's spacing at 20 is 2e-6
        assert bool(((err <= TOL_LOSS) | (err <= U.TAU_LOSS * ref["lscale"])).all()), f"{tag}: loss {float(err.max()):.3g}"
        tidx, got = cpu(ws.tree_idx), cpu(ag.last_loss)
        last = np.array([i for i in range(len(tidx)) if tidx[i] not in tidx[i + 1:]])
        assert_bits_equal(cpu(mem.transitions.tree)[tidx[last]], np.sqrt(got)[last], f"{tag}: priorities")
        _check_gradients(ag, ws, ref, fused, tag, seen)
        _check_optimiser(ag, before, mid, tag)
        if ag.target_tau > 0:
            assert_bits_equal(cpu(mid["target"]), RR.ema_ref(cpu(before["target"]), cpu(mid["flat_param"]), ag.target_tau),
                              f"{tag}: Polyak target")
        else:
            assert torch.equal(after["target"], before["target"]), f"{tag}: the target moves only at a hard copy"
        assert torch.equal(after["target"], mid["target"]), f"{tag}: resets and ReDo leave the target alone"
        since_reset += 1
        for i, (name, st) in enumerate(mids):
            nxt = mids[i + 1][1] if i + 1 < len(mids) else after
            if name == "reset_parameters":
                _check_reset(ag, st, nxt, tag)
                since_reset = 0
            else:
                _check_redo(ag, ws, st, nxt, tag)
        fired = [n for n, _ in mids]
        assert fired == ([n for n, every in (("reset_parameters", ag.reset_interval), ("recycle_dormant", ag.redo_interval))
                          if every and (u + 1) % every == 0]), f"{tag}: passes {fired}"
        if ag._stats is not None:
            rec = ag.learn_stats()
            assert len(rec["loss_mean"]) == 1
            l, w = ref["loss"], ws.weights.double()
            assert abs(float(rec["loss_mean"][0]) - float(l.mean())) <= TOL_LOSS, f"{tag}: learn stats loss_mean"
            assert abs(float(rec["objective"][0]) - float((w * l).mean())) <= TOL_LOSS, f"{tag}: learn stats objective"
            assert_bits_equal(rec["grad_norm"], cpu(opt.grad_norm), f"{tag}: learn stats grad_norm")

    assert set(ag._graphs) == {True, False}, "both captured variants ran"
    names = {k: _kernels(g[0], tmp_path / f"{k}.dot") for k, g in ag._graphs.items()}
    gather, loss, bwd = _expected_kernels(c, ag)
    for pending, ks in names.items():
        own = [k for k in ks if k.startswith("k_")]
        assert own.count(gather) == 1, (pending, own)
        assert own.count(loss) == 1, (pending, own)
        for k in ("k_head_bwd1", "k_head_bwd1_wgrad", "k_head_bwd1_dx"):
            assert own.count(k) == bwd.count(k), (pending, k, own)
        assert own.count("k_head_dh") == own.count("k_head_wgrad2") == int(fused), (pending, own)
        assert own.count("k_noise_factors") == 1 + int(pending), (pending, own)   # the target's draw, and the online one
    print(f"\n{case_id(c)}: kernels {sorted(set(k for k in names[True] if k.startswith('k_')))}; "
          f"max err / scale {', '.join(f'{k} {v:.2e}' for k, v in sorted(seen.items()))}; {ties} near-tied arg-max rows; "
          f"{time.time() - t0:.1f} s")
