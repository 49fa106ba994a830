"""GPU parity tests: the CUDA path (through the C ABI, via the rainbow_b200 host classes) against
 (a) golden vectors recorded from the unmodified reference (tests/golden, oracle/gen_golden.py) and
 (b) the CPU oracle (oracle/rb_oracle.c) on seeded inputs, plus size-independent properties at the
     BASELINE.json sizes (1M-leaf tree, batch 32/512).
Contract: bit-exact for indices, tree sums, uint8/float frames (exact division); float tolerances are
written at each assertion (north star: 1e-5 on the projected distribution and the loss)."""
import argparse
import hashlib
import pickle

import numpy as np
import pytest
import torch

import oracle
from helpers import assert_bits_equal, golden, manifest, oracle_ring_from_golden

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def make_args(**kw):
    d = dict(device=torch.device(DEV), history_length=4, discount=0.99, multi_step=3, priority_weight=0.4,
             priority_exponent=0.5, atoms=51, V_min=-10.0, V_max=10.0, batch_size=32, norm_clip=10.0, model=None,
             learning_rate=6.25e-5, adam_eps=1.5e-4, architecture="canonical", hidden_size=512, noisy_std=0.1)
    d.update(kw)
    return argparse.Namespace(**d)


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def cpu(t):
    return t.detach().cpu().numpy()


def gpu_ring_from_golden(g, pfx, **mem_kw):
    from rainbow_b200.memory import ReplayMemory
    meta = g[pfx + "meta"]
    mem = ReplayMemory(make_args(**mem_kw.pop("args", {})), int(meta[3]), **mem_kw)
    mem.transitions.load_arrays(g[pfx + "sum_tree"], g[pfx + "frames"], g[pfx + "timestep"], g[pfx + "action"],
                                g[pfx + "reward"], g[pfx + "nonterminal"], int(meta[0]), bool(meta[1]), int(meta[2]),
                                float(g[pfx + "max"]))
    mem.t = int(meta[2])
    return mem


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cap", [8, 500, 10000])
def test_tree_update_find_golden(cap):
    from rainbow_b200.memory import SegmentTree
    g = golden("tree")
    t = SegmentTree(cap, DEV)
    ts = t.tree_start
    pri0 = g[f"cap{cap}_pri0"]
    for s in range(0, cap, 64):
        e = min(cap, s + 64)
        t.update(np.arange(s, e) + ts, pri0[s:e])
    assert_bits_equal(t.sum_tree, g[f"cap{cap}_tree0"], "tree0")
    for j in range(4):
        t.update(g[f"cap{cap}_upd{j}_idx"], g[f"cap{cap}_upd{j}_val"])
        assert_bits_equal(t.sum_tree, g[f"cap{cap}_upd{j}_tree"], f"upd{j}")
        assert np.float32(t.max) == g[f"cap{cap}_upd{j}_max"]
    for j in range(3):
        i, v = g[f"cap{cap}_set{j}"]
        t.update(np.array([int(i)]), np.array([v], np.float32))
        assert_bits_equal(t.sum_tree, g[f"cap{cap}_set{j}_tree"], f"set{j}")
    assert np.float32(t.max) == g[f"cap{cap}_final_max"]
    p, di, ti = t.find(g[f"cap{cap}_find_vals"])
    assert_bits_equal(cpu(ti), g[f"cap{cap}_find_tidx"], "tidx")
    assert_bits_equal(cpu(di), g[f"cap{cap}_find_didx"], "didx")
    assert_bits_equal(cpu(p), g[f"cap{cap}_find_probs"], "probs")
    assert int(t._status[0].item()) == 0


@pytest.mark.parametrize("cap", [100000, 1000000])
def test_big_tree_checksums(cap):
    """Full-size (BASELINE.json) trees: checksum of the whole tree and of 4096 descents vs the reference."""
    from rainbow_b200.memory import SegmentTree
    ref = manifest()["big_trees"][str(cap)]
    rs = np.random.RandomState(1)
    t = SegmentTree(cap, DEV)
    ts = t.tree_start
    pri = (rs.uniform(0, 1, cap) ** 0.5 + 1e-3).astype(np.float32)
    for s in range(0, cap, 4096):
        e = min(cap, s + 4096)
        t.update(np.arange(s, e) + ts, pri[s:e])
    for j in range(20):
        idx = rs.randint(0, cap, 32).astype(np.int64) + ts
        val = rs.uniform(0, 2, 32).astype(np.float32)
        t.update(idx, val)
    tree = t.sum_tree
    vals = rs.uniform(0, float(tree[0]), 4096)
    p, di, ti = t.find(vals)
    assert sha(tree) == ref["tree_sha"]
    assert float(tree[0]) == ref["total"] and t.max == ref["max"]
    assert sha(cpu(ti)) == ref["find_tidx_sha"] and sha(cpu(p)) == ref["find_probs_sha"]


def test_tree_update_rejects_bad_index():
    from rainbow_b200.memory import SegmentTree
    t = SegmentTree(64, DEV)
    t.update(np.array([t.tree_start + 3, 5, t.tree_start + 64]), np.array([1.0, 2.0, 3.0], np.float32))
    assert int(t._status[0].item()) == 1
    tree = t.sum_tree
    assert tree[0] == 1.0 and tree[5] == 0.0  # only the valid leaf was written (and propagated)


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", manifest()["replay_cases"], ids=lambda c: c["name"])
def test_replay_sample_golden(case):
    """rb_tree_sample (injected uniforms, all recorded redraws) + rb_gather + rb_tree_update vs the reference."""
    from rainbow_b200 import _lib
    from rainbow_b200.memory import _SampleWorkspace
    g = golden("replay")
    pfx = case["name"] + "_"
    n, B, beta = case["n"], case["B"], case["beta"]
    mem = gpu_ring_from_golden(g, pfx, args=dict(multi_step=n, priority_weight=beta))
    for s in range(6):
        u = g[f"{pfx}s{s}_u01"]
        ws = _SampleWorkspace(B, 4, mem.device)
        mem._launch_sample(ws, u01=torch.from_numpy(u).to(DEV), attempts=u.shape[0])
        st = cpu(ws.status)
        assert st[0] == 1 and st[1] == u.shape[0], "same number of redraws as the reference"
        mem._launch_gather(ws)
        assert_bits_equal(cpu(ws.tree_idx), g[f"{pfx}s{s}_tidx"], "tree idx")
        assert_bits_equal(cpu(ws.states), g[f"{pfx}s{s}_states"], "states")
        assert_bits_equal(cpu(ws.next_states), g[f"{pfx}s{s}_nstates"], "next states")
        assert_bits_equal(cpu(ws.actions), g[f"{pfx}s{s}_actions"], "actions")
        assert_bits_equal(cpu(ws.nonterminals), g[f"{pfx}s{s}_nonterm"], "nonterminals")
        np.testing.assert_allclose(cpu(ws.returns), g[f"{pfx}s{s}_returns"], rtol=0, atol=1e-6)  # f32 dot order
        np.testing.assert_allclose(cpu(ws.weights), g[f"{pfx}s{s}_weights"], rtol=3e-7, atol=0)  # powf: 2 ulp
        # a truncated attempt budget must report an invalid batch instead of looping
        if u.shape[0] > 1:
            ws2 = _SampleWorkspace(B, 4, mem.device)
            mem._launch_sample(ws2, u01=torch.from_numpy(u).to(DEV), attempts=u.shape[0] - 1)
            assert cpu(ws2.status)[0] == 0
        mem.update_priorities(ws.tree_idx, g[f"{pfx}s{s}_raw"])
        assert_bits_equal(mem.transitions.sum_tree, g[f"{pfx}s{s}_tree_after"], "tree after writeback")
        assert np.float32(mem.transitions.max) == g[f"{pfx}s{s}_max_after"]
    it = np.stack([cpu(x) for x, _ in zip(iter(mem), range(12))])
    assert_bits_equal(it, g[pfx + "iter"], "iterator states")


@pytest.mark.parametrize("case", manifest()["replay_cases"][:2], ids=lambda c: c["name"])
def test_replay_numpy_rng_reproduces_reference_stream(case):
    """rng='numpy': same global numpy seed as the generator used -> the reference's exact index sequence."""
    g = golden("replay")
    pfx = case["name"] + "_"
    mem = gpu_ring_from_golden(g, pfx, args=dict(multi_step=case["n"], priority_weight=case["beta"]), rng="numpy")
    np.random.seed(5)
    for s in range(6):
        tidx, states, actions, returns, nstates, nonterm, weights = mem.sample(case["B"])
        assert_bits_equal(cpu(tidx), g[f"{pfx}s{s}_tidx"], "tree idx")
        assert_bits_equal(cpu(states), g[f"{pfx}s{s}_states"], "states")
        mem.update_priorities(cpu(tidx), g[f"{pfx}s{s}_raw"])  # numpy in, like agent.py:100
    assert_bits_equal(mem.transitions.sum_tree, g[f"{pfx}s5_tree_after"], "tree")


def test_append_golden():
    from rainbow_b200.memory import ReplayMemory
    g = golden("append")
    mem = ReplayMemory(make_args(), 8)
    for i in range(19):
        a, r, term = g[f"a{i}_args"]
        state = torch.zeros(4, 84, 84, device=DEV)
        state[-1] = torch.from_numpy(g["last_frames_f32"][i]).to(DEV)
        mem.append(state, int(a), float(r), bool(term))
        if i == 9:
            mem.update_priorities(np.array([mem.transitions.tree_start + 2]), np.array([9.0], np.float32))
        assert_bits_equal(mem.transitions.sum_tree, g[f"a{i}_tree"], f"tree after append {i}")
        assert [mem.transitions.index, int(mem.transitions.full), mem.t] == list(g[f"a{i}_meta"])
        assert list(cpu(mem.transitions.ring_state)[:3]) == list(g[f"a{i}_meta"])
        assert np.float32(mem.transitions.max) == g[f"a{i}_max"]
    d = mem.transitions.data
    assert_bits_equal(d["state"].reshape(8, -1), g["final_frames"], "quantised frames")
    assert_bits_equal(d["timestep"], g["final_timestep"], "timestep")
    assert_bits_equal(d["action"], g["final_action"], "action")
    assert_bits_equal(d["reward"], g["final_reward"], "reward")
    assert_bits_equal(d["nonterminal"].astype(np.uint8), g["final_nonterminal"], "nonterminal")


def test_pickle_roundtrip():
    g = golden("replay")
    mem = gpu_ring_from_golden(g, "c64n3_", args=dict(multi_step=3))
    mem2 = pickle.loads(pickle.dumps(mem))
    assert_bits_equal(mem2.transitions.sum_tree, mem.transitions.sum_tree)
    assert_bits_equal(mem2.transitions.data["state"], mem.transitions.data["state"])
    assert (mem2.transitions.index, mem2.transitions.full, mem2.t) == (mem.transitions.index, mem.transitions.full, mem.t)
    assert list(cpu(mem2.transitions.ring_state)[:3]) == list(cpu(mem.transitions.ring_state)[:3])
    assert mem2.transitions.max == mem.transitions.max
    out = mem2.sample(8)
    assert out[1].shape == (8, 4, 84, 84)


# ------------------------------------------------------------------------------------------------
def synthetic_ring(cap, seed=1, device=DEV, **kw):
    """BASELINE.md synthetic fill (frames on the device to keep it fast), mirrored into an oracle ring
    only for small caps."""
    from rainbow_b200.memory import ReplayMemory
    mem = ReplayMemory(make_args(**kw.pop("args", {})), cap, **kw)
    rs = np.random.RandomState(seed)
    tr = mem.transitions
    timestep = (np.arange(cap) % 1000).astype(np.int32)
    pri = (rs.uniform(0, 1, cap) ** 0.5 + 1e-3).astype(np.float32)
    tr.load_arrays(timestep=timestep, action=rs.randint(0, 6, cap).astype(np.int32),
                   reward=rs.randint(-1, 2, cap).astype(np.float32), nonterminal=(timestep != 999).astype(np.uint8),
                   index=12345 % cap, full=True, t_episode=int(timestep[(12345 % cap) - 1]) + 1)
    gen = torch.Generator(device=device).manual_seed(seed)
    chunk = 65536
    for s in range(0, cap, chunk):
        e = min(cap, s + chunk)
        tr.frames[s:e] = torch.randint(0, 256, (e - s, 7056), dtype=torch.uint8, device=device, generator=gen)
    for s in range(0, cap, 1024):
        e = min(cap, s + 1024)
        tr.update(np.arange(s, e) + tr.tree_start, pri[s:e])
    return mem, pri


@pytest.mark.parametrize("cap,B,n", [(1000000, 32, 3), (1000000, 512, 3), (100000, 32, 20)])
def test_philox_sample_properties_full_size(cap, B, n):
    """Device-RNG sampling at the BASELINE.json sizes, checked through size-independent properties:
    every draw lands in its own stratum (so tree indices are sorted), passes the reference validity test,
    the leaf value returned is the leaf's value, IS weights match the oracle on the same probs, the gather
    matches the oracle gather on the same indices, and two consecutive calls differ."""
    mem, pri = synthetic_ring(cap, args=dict(multi_step=n))
    tr = mem.transitions
    tree = tr.sum_tree
    total = tree[0]
    leaves = tree[tr.tree_start:]
    prefix = np.concatenate([[0.0], np.cumsum(leaves.astype(np.float64))])
    seg = float(np.float32(total) / np.float32(B))
    tidx, states, actions, returns, nstates, nonterm, weights = mem.sample(B)
    mem.check_last_sample()
    tidx_h, probs_h = cpu(tidx), cpu(mem._last.probs)
    didx = tidx_h - tr.tree_start
    assert np.all(np.diff(tidx_h) >= 0), "stratified draws come out sorted"
    assert_bits_equal(probs_h, leaves[didx], "leaf values")
    # stratum k = [k*seg, (k+1)*seg): the leaf's prefix interval must intersect it (float32 tree sums vs the
    # float64 prefix: allow a relative slack of 1e-4 of the total)
    slack = 1e-4 * float(total)
    k = np.arange(B)
    assert np.all(prefix[didx + 1] >= k * seg - slack) and np.all(prefix[didx] <= (k + 1) * seg + slack)
    assert oracle.batch_valid(didx, probs_h, tr.index, cap, n, 4)
    np.testing.assert_allclose(cpu(weights), oracle.is_weights(probs_h, total, cap, 0.4), rtol=3e-7)
    # gather vs oracle gather on the same indices (only the touched records are mirrored to the host)
    H = 4
    win = (didx[:, None] + np.arange(-H + 1, n + 1)[None, :]) % cap
    uniq, inv = np.unique(win, return_inverse=True)
    ot = oracle.OracleTree(max(2, uniq.size + (uniq.size % 2)))
    sel = torch.as_tensor(uniq, device=DEV)
    ot.frames[:uniq.size] = cpu(tr.frames[sel])
    ot.timestep[:uniq.size] = cpu(tr.timestep[sel])
    ot.action[:uniq.size] = cpu(tr.action[sel])
    ot.reward[:uniq.size] = cpu(tr.reward[sel])
    ot.nonterminal[:uniq.size] = cpu(tr.nonterminal[sel])
    # run the oracle gather sample by sample on a compacted ring: window record j of sample b sits at inv[b, j]
    inv = inv.reshape(win.shape)
    gam = np.array([0.99 ** i for i in range(n)], np.float32)
    for b in range(0, B, max(1, B // 16)):
        mini = oracle.OracleTree(2 * (H + n))
        rows = inv[b]
        mini.frames[:H + n] = ot.frames[rows]
        mini.timestep[:H + n] = ot.timestep[rows]
        mini.action[:H + n] = ot.action[rows]
        mini.reward[:H + n] = ot.reward[rows]
        mini.nonterminal[:H + n] = ot.nonterminal[rows]
        mini.timestep[H + n:] = 1  # padding records never start an episode
        o_s, o_a, o_r, o_ns, o_nt = oracle.gather(mini, np.array([H - 1]), H, n, gam)
        assert_bits_equal(cpu(states[b]), o_s[0], "states")
        assert_bits_equal(cpu(nstates[b]), o_ns[0], "next states")
        assert int(actions[b]) == int(o_a[0]) and float(nonterm[b, 0]) == float(o_nt[0, 0])
        assert_bits_equal(cpu(returns[b:b + 1]), o_r, "returns")
    tidx2 = cpu(mem.sample(B)[0])
    assert not np.array_equal(tidx2, tidx_h), "the device counter advances between calls"


def test_tree_invariant_after_many_updates_full_size():
    """1M-leaf tree: after 200 batched write-backs every internal node equals fl32(left+right) of its
    children, the root equals the oracle's root for the same update stream, and max is monotone."""
    mem, pri = synthetic_ring(1000000)
    tr = mem.transitions
    ot = oracle.OracleTree(1000000, with_data=False)
    ot.sum_tree[:] = tr.sum_tree
    ot.max[0] = tr.max
    rs = np.random.RandomState(3)
    for it in range(200):
        B = 32 if it % 4 else 512
        idx = rs.randint(0, 1000000, B).astype(np.int64) + tr.tree_start
        if it % 3 == 0:
            idx[B // 2:] = idx[:B - B // 2]  # duplicates
        raw = rs.uniform(0, 4, B).astype(np.float32)
        mem.update_priorities(idx, raw)
        ot.update(idx, oracle.pow_priorities(raw, 0.5))
    tree = tr.sum_tree
    assert_bits_equal(tree, ot.sum_tree, "1M tree after 200 updates")
    assert tr.max == float(ot.max[0])
    ts = tr.tree_start
    n_int = (tree.size - 1) // 2  # nodes whose two children exist
    par = np.arange(n_int)
    touched = tree[par] != 0
    assert np.array_equal(tree[par][touched], (tree[2 * par + 1] + tree[2 * par + 2])[touched])


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", manifest()["learn_cases"], ids=lambda c: c["name"])
def test_c51_golden(case):
    from rainbow_b200.agent import c51_loss_grad
    g = golden("learn")
    p = case["name"] + "_"
    B, A, Z = case["B"], case["A"], case["Z"]
    d = lambda k: torch.from_numpy(np.ascontiguousarray(g[p + k])).to(DEV)
    m = torch.empty(B, Z, device=DEV)
    astar = torch.empty(B, dtype=torch.int64, device=DEV)
    gamma_n = case["discount"] ** case["n"]
    loss, grad = c51_loss_grad(d("q_s"), d("q_ns"), d("q_t"), d("actions"), d("returns"), d("nonterm"), d("weights"),
                               d("support"), case["V_min"], case["V_max"], case["delta_z"], gamma_n, m_out=m,
                               astar_out=astar)
    assert np.array_equal(cpu(astar), g[p + "astar"])
    # north star: within 1e-5 on the projected distribution and the loss
    np.testing.assert_allclose(cpu(m), g[p + "m"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(cpu(loss), g[p + "loss"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(cpu(grad), g[p + "grad"], rtol=0, atol=1e-6)
    # and against the oracle on the same inputs: same op order, so only exp/log ulps differ
    o_loss, o_grad, o_m, o_astar = oracle.c51(g[p + "q_s"], g[p + "q_ns"], g[p + "q_t"], g[p + "actions"],
                                               g[p + "returns"], g[p + "nonterm"], g[p + "weights"], g[p + "support"],
                                               case["V_min"], case["V_max"], case["delta_z"], gamma_n)
    np.testing.assert_allclose(cpu(m), o_m, rtol=0, atol=1e-6)
    np.testing.assert_allclose(cpu(loss), o_loss, rtol=2e-6, atol=2e-6)


def test_c51_batch512_oracle():
    """BASELINE config C4 shape (B=512, A=6, Z=51) on seeded logits vs the oracle."""
    from rainbow_b200.agent import c51_loss_grad
    rs = np.random.RandomState(0)
    B, A, Z = 512, 6, 51
    q = [rs.normal(0, 2, (B, A, Z)).astype(np.float32) for _ in range(3)]
    actions = rs.randint(0, A, B).astype(np.int64)
    returns = (rs.randint(-1, 2, (B, 3)).astype(np.float32) @ np.array([1, 0.99, 0.99 ** 2], np.float32))
    nonterm = (rs.uniform(size=(B, 1)) > 0.1).astype(np.float32)
    w = rs.uniform(0.1, 1, B).astype(np.float32)
    support = cpu(torch.linspace(-10, 10, Z))
    dz, gn = 20 / 50, 0.99 ** 3
    t = lambda a: torch.from_numpy(a).to(DEV)
    m = torch.empty(B, Z, device=DEV)
    loss, grad = c51_loss_grad(t(q[0]), t(q[1]), t(q[2]), t(actions), t(returns), t(nonterm), t(w), t(support), -10.0,
                               10.0, dz, gn, m_out=m)
    o_loss, o_grad, o_m, _ = oracle.c51(q[0], q[1], q[2], actions, returns, nonterm, w, support, -10.0, 10.0, dz, gn)
    np.testing.assert_allclose(cpu(m), o_m, rtol=0, atol=1e-6)
    np.testing.assert_allclose(cpu(loss), o_loss, rtol=2e-6, atol=2e-6)
    np.testing.assert_allclose(cpu(grad), o_grad, rtol=0, atol=1e-7)
    np.testing.assert_allclose(cpu(m).sum(1), 1.0, atol=1e-5)


# ------------------------------------------------------------------------------------------------
def test_noise_injected_golden():
    from rainbow_b200.model import NoisyLinear, resample_noise
    g = golden("noise")
    names = ("l37x19", "l576x64", "l512x51")
    layers = [NoisyLinear(int(n[1:].split("x")[0]), int(n.split("x")[1])).to(DEV) for n in names]
    x_in = torch.from_numpy(np.concatenate([g[n + "_x_in"] for n in names])).to(DEV)
    x_out = torch.from_numpy(np.concatenate([g[n + "_x_out"] for n in names])).to(DEV)
    ctr = torch.zeros(1, dtype=torch.int64, device=DEV)
    resample_noise(layers, 1, ctr, x_in, x_out)
    for n, layer in zip(names, layers):
        o_w, o_b = oracle.noisy(g[n + "_x_in"], g[n + "_x_out"])
        assert_bits_equal(cpu(layer.weight_epsilon), o_w, "weight_epsilon vs oracle")
        assert_bits_equal(cpu(layer.bias_epsilon), o_b, "bias_epsilon vs oracle")
        # vs the reference: its sqrt goes through MKL VML (1 ulp), see tests/test_oracle_golden.py
        np.testing.assert_allclose(cpu(layer.weight_epsilon), g[n + "_w_eps"], rtol=4e-7, atol=0)
        np.testing.assert_allclose(cpu(layer.bias_epsilon), g[n + "_b_eps"], rtol=1.3e-7, atol=0)
    assert int(ctr.item()) == 0, "injected mode leaves the counter alone"


def test_noise_philox_statistics():
    """Device draws: rank-1 structure, f(x) moments of a standard normal, fresh numbers per call."""
    from rainbow_b200.model import DQN
    net = DQN(make_args(), 6).to(DEV)
    net.reset_noise()
    sd = net.state_dict()                     # weight_epsilon / bias_epsilon are materialised lazily, on inspection
    w1 = cpu(sd["fc_h_v.weight_epsilon"]).copy()
    b1 = cpu(sd["fc_h_v.bias_epsilon"]).copy()
    # rank 1: W[o, i] == b[o] * e_in[i] with e_in recovered from one row
    o0 = int(np.argmax(np.abs(b1)))
    e_in = w1[o0] / b1[o0]
    np.testing.assert_allclose(w1, np.outer(b1, e_in), rtol=1e-5, atol=1e-7)
    # |f(x)| = sqrt|x| : E = 0.822, E f^2 = E|x| = 0.798 ; sign symmetric
    allv = np.concatenate([cpu(l.bias_epsilon) for l in net.noisy_layers()] + [e_in])
    assert abs(np.mean(allv)) < 0.05
    assert abs(np.mean(allv ** 2) - 0.7979) < 0.05
    assert abs(np.mean(np.abs(allv)) - 0.8222) < 0.04
    x = np.sign(allv) * allv ** 2  # invert f: should be standard normal
    assert abs(np.std(x) - 1.0) < 0.05 and abs(np.mean(x ** 4) - 3.0) < 0.5
    net.reset_noise()
    assert not np.array_equal(cpu(net.state_dict()["fc_h_v.weight_epsilon"]), w1)
    assert int(net._noise_counter.item()) == 2
    # layers do not share draws
    assert not np.array_equal(cpu(net.fc_h_a.bias_epsilon), cpu(net.fc_h_v.bias_epsilon))


def test_clip_adam_oracle():
    from rainbow_b200 import _lib
    L = _lib.load()
    rs = np.random.RandomState(0)
    P = 100003 * 4
    p = rs.normal(0, 0.1, P).astype(np.float32)
    m = np.zeros(P, np.float32)
    v = np.zeros(P, np.float32)
    dp, dm, dv = (torch.from_numpy(a.copy()).to(DEV) for a in (p, m, v))
    step = torch.zeros(1, dtype=torch.int64, device=DEV)
    part = torch.zeros(L.rb_clip_adam_scratch_elems(), dtype=torch.float64, device=DEV)
    norm = torch.zeros(1, device=DEV)
    for it in range(1, 6):
        scale = 30.0 if it % 2 else 0.01  # with and without clipping
        g = (rs.normal(0, 1, P) * scale / np.sqrt(P)).astype(np.float32)
        dg = torch.from_numpy(g).to(DEV)
        _lib.check(L.rb_clip_adam(dp.data_ptr(), dg.data_ptr(), dm.data_ptr(), dv.data_ptr(), P, 1.0, 10.0, 6.25e-5,
                                  0.9, 0.999, 1.5e-4, step.data_ptr(), part.data_ptr(), norm.data_ptr(), None,
                                  torch.cuda.current_stream().cuda_stream))
        o_norm = oracle.clip_adam(p, g.copy(), m, v, 10.0, 6.25e-5, 0.9, 0.999, 1.5e-4, it)
        assert abs(float(norm.item()) - o_norm) <= 2e-6 * o_norm
        assert int(step.item()) == it
        np.testing.assert_allclose(cpu(dm), m, rtol=1e-5, atol=1e-9)
        np.testing.assert_allclose(cpu(dv), v, rtol=1e-5, atol=1e-12)
        np.testing.assert_allclose(cpu(dp), p, rtol=0, atol=2e-7)


# ------------------------------------------------------------------------------------------------
class FakeEnv:
    def __init__(self, a):
        self.a = a

    def action_space(self):
        return self.a


@pytest.mark.parametrize("fused,cudnn", [(True, True), (True, False), (False, True)],
                         ids=["fused_head_manual_conv_bwd", "fused_head_autograd_convs", "library_gemm_head"])
def test_learner_step_vs_reference_golden(fused, cudnn):
    """End to end: one Agent.learn on a tiny data-efficient net vs the unmodified reference CPU run
    (tests/golden/model_step.npz): same initial weights, same batch, same target-net noise draw.
    GPU conv/GEMM (fp32, TF32 off) vs CPU conv/GEMM: loss within 1e-5, gradients within 1e-6 abs."""
    from rainbow_b200.agent import Agent
    g = golden("model_step")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    B, A = 4, 3
    args = make_args(batch_size=B, architecture="data-efficient", hidden_size=64, multi_step=3, cuda_graph=False, fused_head=fused)
    ag = Agent(args, FakeEnv(A))
    sd0 = {k[4:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("sd0.")}
    ag.online_net.load_state_dict(sd0)
    ag.update_target_net()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    states = t(g["states_u8"]).float() / 255
    nstates = t(g["nstates_u8"]).float() / 255
    batch = (torch.arange(B, device=DEV), states, t(g["actions"]), t(g["returns"]), nstates, t(g["nonterm"]),
             t(g["weights"]))
    # target noise: randn order is eps_in, eps_out per layer (model.py:37-38), layers in reset order
    x_in = t(np.concatenate([g[f"target_randn{2 * i}"] for i in range(4)]))
    x_out = t(np.concatenate([g[f"target_randn{2 * i + 1}"] for i in range(4)]))
    assert ag._fused_path(B) == fused
    with torch.backends.cudnn.flags(enabled=cudnn, allow_tf32=False):   # cuDNN off (main.py's default) -> convs go through autograd
        assert ag.online_net.manual_conv_ok(states) == cudnn
        loss = ag._update_from_batch(batch, target_noise=(x_in, x_out))
    np.testing.assert_allclose(cpu(loss), g["loss"], rtol=1e-5, atol=1e-5)
    for k, p in ag.online_net.named_parameters():
        # clip_grad_norm_ scales .grad in place in the reference when norm > 10; here the norm is < 10
        np.testing.assert_allclose(cpu(p.grad), g["grad." + k], rtol=0, atol=1e-6, err_msg=k)
    for k, v in ag.target_net.state_dict().items():
        if "epsilon" in k:
            np.testing.assert_allclose(cpu(v), g["target_eps." + k], rtol=4e-7, atol=0)
    # parameters after clip+Adam.  First Adam step moves every weight by ~lr*g/(|g|+eps): compare the UPDATE
    # with an absolute tolerance of 2% of lr (gradients near zero are the sensitive ones)
    lr = args.learning_rate
    for k, p in ag.online_net.named_parameters():
        np.testing.assert_allclose(cpu(p), g["sd1." + k], rtol=0, atol=0.02 * lr, err_msg=k)


# ------------------------------------------------------------------------------------------------
# fused noisy dueling head (csrc/rb_head.cu) against the library path (composed weights + F.linear + autograd)
def _head_net(arch="canonical", hidden=512, actions=6, seed=0):
    from rainbow_b200.model import DQN
    torch.manual_seed(seed)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    net = DQN(make_args(architecture=arch, hidden_size=hidden), actions).to(DEV)
    with torch.no_grad():  # make sigma non-trivial so the noise terms matter
        for m in net.noisy_layers():
            m.weight_sigma.mul_(torch.empty_like(m.weight_sigma).uniform_(0.5, 3.0))
            m.bias_sigma.mul_(torch.empty_like(m.bias_sigma).uniform_(0.5, 3.0))
    net.reset_noise()
    return net


def _library_head(net, feats):
    """Reference formulation on the GPU: materialised weight_epsilon, composed weights, F.linear (model.py:42-44,73-75)."""
    import torch.nn.functional as F
    net.materialise_noise()
    v = net.fc_z_v(F.relu(net.fc_h_v(feats)))
    a = net.fc_z_a(F.relu(net.fc_h_a(feats)))
    return v, a


@pytest.mark.parametrize("arch,hidden,actions", [("canonical", 512, 6), ("data-efficient", 256, 18), ("data-efficient", 64, 3)])
@pytest.mark.parametrize("rows", [1, 32, 64, 100])
def test_fused_head_forward(arch, hidden, actions, rows):
    net = _head_net(arch, hidden, actions)
    feats = torch.randn(rows, net.conv_output_size, device=DEV).relu()
    with torch.no_grad():
        for mode in ("train", "eval"):
            getattr(net, mode)()
            v, a = _library_head(net, feats)
            q_ref = v.view(rows, 1, -1) + a.view(rows, actions, -1) - a.view(rows, actions, -1).mean(1, keepdim=True)
            z, h, p = net.head().forward(feats[:rows // 2 + 1].contiguous(), feats[rows // 2 + 1:].contiguous() if rows > 1 else None)
            q = net.head().logits(z)
            np.testing.assert_allclose(cpu(z), cpu(torch.cat([v, a], 1)), rtol=1e-4, atol=2e-5)
            assert int(net.head()._tickets.abs().sum()) == 0, "split-K tickets are self-resetting"
            np.testing.assert_allclose(cpu(q), cpu(q_ref), rtol=1e-4, atol=2e-5)
            import torch.nn.functional as F
            h_ref = torch.cat([F.relu(net.fc_h_v(feats)), F.relu(net.fc_h_a(feats))], 1)
            np.testing.assert_allclose(cpu(h), cpu(h_ref), rtol=1e-4, atol=2e-5)
    net.train()
    x = torch.rand(3, 4, 84, 84, device=DEV)
    with torch.no_grad():
        q_f = net.logits(x)                       # fused inference path (what Agent.act uses)
        net.use_fused_head = False
        q_l = net.logits(x)
    np.testing.assert_allclose(cpu(q_f), cpu(q_l), rtol=1e-4, atol=2e-5)


@pytest.mark.parametrize("arch,hidden,actions", [("canonical", 512, 6), ("data-efficient", 256, 6), ("data-efficient", 64, 3)])
@pytest.mark.parametrize("m_lo,m_hi", [(32, 32), (32, 0), (16, 16), (8, 0), (1, 0), (40, 60), (20, 0)])
def test_fused_head_layer1_tensor_core(arch, hidden, actions, m_lo, m_hi):
    """Layer 1 on the tensor cores (csrc/rb_head_tc.cu: TMA + wgmma, error-compensated TF32) against the composed-weight
    fp32 library GEMM (model.py:42-44) and against the FFMA kernel: fp32-equivalent results (<= 2e-5 of the tensor's scale,
    the same bound the FFMA kernel is held to; observed ~1e-6), in training and eval mode, ragged row counts included."""
    import torch.nn.functional as F
    from rainbow_b200 import _lib
    L = _lib.load()
    net = _head_net(arch, hidden, actions)
    torch.manual_seed(3)
    x_lo = torch.randn(m_lo, net.conv_output_size, device=DEV).relu()
    x_hi = torch.randn(m_hi, net.conv_output_size, device=DEV).relu() if m_hi else None
    feats = x_lo if x_hi is None else torch.cat([x_lo, x_hi])
    with torch.no_grad():
        for mode in ("train", "eval"):
            getattr(net, mode)()
            h_ref = torch.cat([F.relu(net.fc_h_v(feats)), F.relu(net.fc_h_a(feats))], 1) if mode == "eval" else None
            if mode == "train":
                net.materialise_noise()
                h_ref = torch.cat([F.relu(net.fc_h_v(feats)), F.relu(net.fc_h_a(feats))], 1)
            v, a = _library_head(net, feats)
            try:
                L.rb_head_debug(4)                                   # FFMA layer 1
                z_ff, h_ff, _ = net.head().forward(x_lo, x_hi)
                z_ff, h_ff = z_ff.clone(), h_ff.clone()
            finally:
                L.rb_head_debug(0)
            z, h, _ = net.head().forward(x_lo, x_hi)                 # tensor-core layer 1 (default)
            z, h = z.clone(), h.clone()
            np.testing.assert_allclose(cpu(h), cpu(h_ref), rtol=1e-4, atol=2e-5)
            np.testing.assert_allclose(cpu(h), cpu(h_ff), rtol=1e-4, atol=2e-5)
            np.testing.assert_allclose(cpu(z), cpu(torch.cat([v, a], 1)), rtol=1e-4, atol=2e-5)
            z2, h2, _ = net.head().forward(x_lo, x_hi)               # deterministic: bit-identical on a second launch
            assert torch.equal(h2, h) and torch.equal(z2, z)
    net.train()


def test_noise_factors_plus_outer_equals_resample():
    from rainbow_b200.model import resample_noise
    net = _head_net()
    ctr0 = int(net._noise_counter.item())
    net.materialise_noise()
    w_fact = [cpu(m.weight_epsilon).copy() for m in net.noisy_layers()]
    b_fact = [cpu(m.bias_epsilon).copy() for m in net.noisy_layers()]
    ctr = torch.tensor([ctr0 - 1], dtype=torch.int64, device=DEV)     # the draw reset_noise() consumed
    resample_noise(net.noisy_layers(), net.noise_seed, ctr)            # K6 with the same seed / counter
    for m, w, b in zip(net.noisy_layers(), w_fact, b_fact):
        assert_bits_equal(cpu(m.weight_epsilon), w, "weight_epsilon")
        assert_bits_equal(cpu(m.bias_epsilon), b, "bias_epsilon")
    # state_dict() materialises, load_state_dict() recovers the factors (to rounding)
    net.reset_noise()
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    f_in, f_out = net._f_in.clone(), net._f_out.clone()
    net.reset_noise()
    net.load_state_dict(sd)
    np.testing.assert_allclose(cpu(net._f_out), cpu(f_out), rtol=0, atol=0)
    np.testing.assert_allclose(cpu(net._f_in), cpu(f_in), rtol=3e-7, atol=1e-9)


@pytest.mark.parametrize("arch,hidden,actions,B", [("canonical", 512, 6, 32), ("data-efficient", 256, 4, 17), ("data-efficient", 64, 3, 1)])
def test_fused_head_backward(arch, hidden, actions, B):
    net = _head_net(arch, hidden, actions, seed=1)
    K1, Z = net.conv_output_size, net.atoms
    feats = torch.randn(B, K1, device=DEV).relu().requires_grad_(True)
    dz = torch.randn(B, Z * (1 + actions), device=DEV) * 0.1
    v, a = _library_head(net, feats)
    out = torch.cat([v, a], 1)
    params = [p for m in net.noisy_layers() for p in (m.weight_mu, m.weight_sigma, m.bias_mu, m.bias_sigma)]
    ref = torch.autograd.grad(out, [feats] + params, dz)
    for p in params:
        p.grad = torch.full_like(p, 123.0)       # must be overwritten, not accumulated
    with torch.no_grad():
        z, h, p_ = net.head().forward(feats.detach())
        dh = torch.empty(B + 32, 2 * hidden, device=DEV)   # dh [B][2H], then dhT [2H][32]
        dx = torch.empty(B, K1, device=DEV)
        net.head().backward(p_, feats.detach(), h[:B], dz, dh, dx)
    scale = lambda t: float(t.abs().max()) + 1e-12
    np.testing.assert_allclose(cpu(dx), cpu(ref[0]), rtol=0, atol=2e-5 * scale(ref[0]))
    for p, r in zip(params, ref[1:]):
        np.testing.assert_allclose(cpu(p.grad), cpu(r), rtol=0, atol=2e-5 * scale(r))


@pytest.mark.parametrize("actions,B", [(6, 32), (18, 5)])
def test_c51_dueling_entry(actions, B):
    """rb_c51_dueling_loss_grad (fed by head partials) == rb_c51_loss_grad on the assembled logits, and its dz is
    the dueling-combine backward of the logit gradient."""
    from rainbow_b200.agent import c51_dueling_loss_grad, c51_loss_grad
    on, tg = _head_net("data-efficient", 128, actions, seed=2), _head_net("data-efficient", 128, actions, seed=3)
    K1, Z, A = on.conv_output_size, on.atoms, actions
    rs = np.random.RandomState(0)
    x = torch.randn(2 * B, K1, device=DEV).relu() * 3
    t = lambda a: torch.from_numpy(a).to(DEV)
    acts = t(rs.randint(0, A, B).astype(np.int64))
    rets = t(rs.uniform(-2, 2, B).astype(np.float32))
    nont = t((rs.uniform(size=(B, 1)) > 0.2).astype(np.float32))
    w = t(rs.uniform(0.2, 1, B).astype(np.float32))
    support = torch.linspace(-10, 10, Z).to(DEV)
    with torch.no_grad():
        z_on, _, _ = on.head().forward(x[:B].contiguous(), x[B:].contiguous())
        z_t, _, _ = tg.head().forward(x[B:].contiguous())
        q_on = on.head().logits(z_on)
        q_t = tg.head().logits(z_t)
        m1 = torch.empty(B, Z, device=DEV); m2 = torch.empty(B, Z, device=DEV)
        a1 = torch.empty(B, dtype=torch.int64, device=DEV); a2 = torch.empty(B, dtype=torch.int64, device=DEV)
        loss_ref, gq = c51_loss_grad(q_on[:B].contiguous(), q_on[B:].contiguous(), q_t, acts, rets, nont, w, support, -10.0, 10.0,
                                     0.4, 0.99 ** 3, m_out=m1, astar_out=a1)
        loss, dz = c51_dueling_loss_grad(z_on, z_t, A, Z, acts, rets, nont, w, support, -10.0, 10.0, 0.4, 0.99 ** 3,
                                         m_out=m2, astar_out=a2)
    assert torch.equal(a1, a2)
    np.testing.assert_allclose(cpu(m2), cpu(m1), rtol=0, atol=1e-6)
    np.testing.assert_allclose(cpu(loss), cpu(loss_ref), rtol=1e-5, atol=1e-5)
    dzv_ref = gq.sum(1)                                            # q = zv + za - mean_a za
    dza_ref = gq - gq.mean(1, keepdim=True)
    np.testing.assert_allclose(cpu(dz[:, :Z]), cpu(dzv_ref), rtol=1e-5, atol=1e-8)
    np.testing.assert_allclose(cpu(dz[:, Z:]).reshape(B, A, Z), cpu(dza_ref), rtol=1e-5, atol=1e-8)


def test_agent_learn_graph_and_eager():
    """The whole update as a CUDA graph: runs, keeps the tree consistent, moves the weights, and exposes
    the same API surface main.py / test.py use."""
    from rainbow_b200.agent import Agent
    torch.manual_seed(0)
    for use_graph in (False, True):
        args = make_args(cuda_graph=use_graph, architecture="data-efficient", hidden_size=64, batch_size=16)
        mem, _ = synthetic_ring(4096, args=dict())
        ag = Agent(args, FakeEnv(6))
        w0 = ag.optimiser.flat_param.clone()
        tree0 = mem.transitions.sum_tree.copy()
        for it in range(12):
            mem.priority_weight = min(mem.priority_weight + 0.01, 1.0)  # main.py:161
            ag.reset_noise()
            ag.learn(mem)
        mem.check_last_sample()
        assert (ag._graph is not None) == use_graph
        assert int(ag.optimiser.step_count.item()) == 12
        assert torch.isfinite(ag.last_loss).all()
        assert not torch.equal(w0, ag.optimiser.flat_param)
        tree = mem.transitions.sum_tree
        assert not np.array_equal(tree, tree0)
        ts = mem.transitions.tree_start
        par = np.arange((tree.size - 1) // 2)
        assert np.array_equal(tree[par], tree[2 * par + 1] + tree[2 * par + 2]), "sum-tree invariant"
        assert abs(float(mem._beta_dev.item()) - mem.priority_weight) < 1e-6
        # API used by main.py / test.py
        state = next(iter(mem))
        a = ag.act(state)
        assert 0 <= a < 6 and isinstance(ag.evaluate_q(state), float)
        ag.eval(); ag.act_e_greedy(state); ag.train(); ag.update_target_net()
        for (k1, v1), (k2, v2) in zip(ag.online_net.state_dict().items(), ag.target_net.state_dict().items()):
            assert k1 == k2 and torch.equal(v1, v2)


def test_state_dict_keys_match_reference_layout():
    from rainbow_b200.model import DQN
    net = DQN(make_args(), 6)
    keys = set(net.state_dict().keys())
    want = {f"convs.{i}.{k}" for i in (0, 2, 4) for k in ("weight", "bias")}
    want |= {f"fc_{l}.{k}" for l in ("h_v", "h_a", "z_v", "z_a")
             for k in ("weight_mu", "weight_sigma", "bias_mu", "bias_sigma", "weight_epsilon", "bias_epsilon")}
    assert keys == want
