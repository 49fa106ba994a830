#!/usr/bin/env python
"""Generate golden vectors from the UNMODIFIED reference (Kaixhin/Rainbow).

Runs only in the build container (needs /root/reference, read-only).  It imports
the reference's memory.py / model.py / agent.py as they are, drives them through
their public methods with a fake `args` namespace and a fake env, and records
inputs/outputs as small .npz fixtures under tests/golden/.  Randomness the
reference draws internally (np.random.uniform in memory.py:129, torch.randn in
model.py:33) is RECORDED by wrapping those library functions in this harness --
the reference files are never edited or copied.

    python oracle/gen_golden.py            # writes tests/golden/*.npz + MANIFEST.json
    python oracle/gen_golden.py ref_pickle_state   # only tests/golden/ref_pickle_state.json
    python oracle/gen_golden.py replay_history     # only tests/golden/replay_history.npz + its MANIFEST.json key

Versions are recorded in MANIFEST.json (numpy/torch behaviour is the effective
pin: the reference's requirements.txt pins nothing).
"""
import argparse
import hashlib
import json
import os
import sys

import numpy as np
import torch

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")

sys.path.insert(0, REF)
import agent as ref_agent  # noqa: E402
import memory as ref_memory  # noqa: E402
import model as ref_model  # noqa: E402


def make_args(**kw):
    d = dict(device=torch.device("cpu"), history_length=4, discount=0.99, multi_step=3, priority_weight=0.4,
             priority_exponent=0.5, atoms=51, V_min=-10.0, V_max=10.0, batch_size=32, norm_clip=10.0, model=None,
             learning_rate=6.25e-5, adam_eps=1.5e-4, architecture="canonical", hidden_size=512, noisy_std=0.1)
    d.update(kw)
    return argparse.Namespace(**d)


class FakeEnv:
    def __init__(self, a):
        self.a = a

    def action_space(self):
        return self.a


def bare_tree(size):
    """SegmentTree without the 4-minute Python-list data constructor (memory.py:19): build the object
    field by field in the harness; every METHOD used afterwards is the reference's own."""
    t = ref_memory.SegmentTree.__new__(ref_memory.SegmentTree)
    t.index = 0
    t.size = size
    t.full = False
    t.tree_start = 2 ** (size - 1).bit_length() - 1
    t.sum_tree = np.zeros((t.tree_start + size,), dtype=np.float32)
    t.data = None
    t.max = 1
    return t


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


# --------------------------------------------------------------------------------------------
def gen_tree():
    """SegmentTree.update / _update_index / find on trees of several sizes."""
    out = {}
    rs = np.random.RandomState(7)
    for cap in (8, 500, 10000):
        t = bare_tree(cap)
        ts = t.tree_start
        # op 0: all leaves through update() in chunks of 64 (memory.py:44-48)
        pri0 = (rs.uniform(0, 1, cap) ** 0.5 + 1e-3).astype(np.float32)
        for s in range(0, cap, 64):
            e = min(cap, s + 64)
            t.update(np.arange(s, e) + ts, pri0[s:e])
        out[f"cap{cap}_pri0"] = pri0
        out[f"cap{cap}_tree0"] = t.sum_tree.copy()
        # op 1..4: batches with duplicates
        for j in range(4):
            B = (4, 32, 32, 512)[j] if cap >= 500 else (4, 8, 8, 8)[j]
            idx = rs.randint(0, cap, B).astype(np.int64)
            if j >= 1:
                idx[B // 2:] = idx[: B - B // 2]  # force duplicates: later entries must win
            idx = rs.permutation(idx) + ts
            val = rs.uniform(0, 3, B).astype(np.float32)
            if j == 3:
                val[::5] = 0.0  # zero priorities too
            t.update(idx, val)
            out[f"cap{cap}_upd{j}_idx"] = idx
            out[f"cap{cap}_upd{j}_val"] = val
            out[f"cap{cap}_upd{j}_tree"] = t.sum_tree.copy()
            out[f"cap{cap}_upd{j}_max"] = np.float32(t.max)
        # single-leaf walks (memory.py:51-54)
        for j in range(3):
            i = int(rs.randint(0, cap)) + ts
            v = np.float32(rs.uniform(0, 5))
            t._update_index(i, v)
            out[f"cap{cap}_set{j}"] = np.array([i, v], dtype=np.float64)
            out[f"cap{cap}_set{j}_tree"] = t.sum_tree.copy()
        out[f"cap{cap}_final_max"] = np.float32(t.max)
        # find(): edge values (memory.py:64-82)
        total = float(t.sum_tree[0])
        pref = np.cumsum(t.sum_tree[ts:ts + cap].astype(np.float64))
        edge = [0.0, total, total * 2, np.nextafter(total, 0), np.nextafter(total, np.inf), 1e-30]
        for k in rs.randint(0, cap - 1, 6):
            edge += [pref[k], np.nextafter(pref[k], 0), np.nextafter(pref[k], np.inf)]
        vals = np.concatenate([np.array(edge, np.float64), rs.uniform(0, total, 200)])
        p, di, ti = t.find(vals)
        out[f"cap{cap}_find_vals"] = vals
        out[f"cap{cap}_find_probs"] = p
        out[f"cap{cap}_find_didx"] = di.astype(np.int64)
        out[f"cap{cap}_find_tidx"] = ti.astype(np.int64)
    np.savez_compressed(os.path.join(OUT, "tree.npz"), **out)

    # big trees: checksums only (size-independent pin for 100k / 1M)
    big = {}
    for cap in (100000, 1000000):
        rs = np.random.RandomState(1)
        t = bare_tree(cap)
        ts = t.tree_start
        pri = (rs.uniform(0, 1, cap) ** 0.5 + 1e-3).astype(np.float32)
        for s in range(0, cap, 4096):
            e = min(cap, s + 4096)
            t.update(np.arange(s, e) + ts, pri[s:e])
        for j in range(20):
            idx = rs.randint(0, cap, 32).astype(np.int64) + ts
            val = rs.uniform(0, 2, 32).astype(np.float32)
            t.update(idx, val)
        vals = rs.uniform(0, float(t.sum_tree[0]), 4096)
        p, di, ti = t.find(vals)
        big[str(cap)] = dict(tree_sha=sha(t.sum_tree), total=float(t.sum_tree[0]), max=float(t.max),
                             find_tidx_sha=sha(ti.astype(np.int64)), find_probs_sha=sha(p))
    return big


# --------------------------------------------------------------------------------------------
class UniformRecorder:
    """Wraps np.random.uniform (called at memory.py:129) and records the unit uniforms behind each call."""

    def __init__(self):
        self.calls = []
        self.orig = np.random.uniform

    def __enter__(self):
        def wrapped(low, high, size):
            st = np.random.get_state()
            res = self.orig(low, high, size)
            rs = np.random.RandomState()
            rs.set_state(st)
            u = rs.random_sample(size)
            assert np.array_equal(res, low + (float(high) - low) * u)
            self.calls.append(u.copy())
            return res

        np.random.uniform = wrapped
        return self

    def __exit__(self, *a):
        np.random.uniform = self.orig


def pattern_state(i):
    """Synthetic [4,84,84] float state whose last frame is a compressible pattern covering all 256 levels."""
    pix = np.arange(84 * 84, dtype=np.int64)
    lvl = ((pix * (2 * (i % 5) + 1) + 13 * i) % 256).astype(np.float32)
    f = torch.zeros(4, 84, 84)
    f[-1] = torch.from_numpy(lvl.reshape(84, 84)) / 255  # values k/255: mul(255)+truncate hits both k and k-1
    if i % 3 == 0:
        f[-1] += 0.0009  # and some mid-bucket values
        f[-1].clamp_(0, 1)
    return f


def dump_ring(mem, out, prefix):
    t = mem.transitions
    out[prefix + "sum_tree"] = t.sum_tree.copy()
    out[prefix + "frames"] = t.data["state"].reshape(t.size, -1).copy()
    out[prefix + "timestep"] = t.data["timestep"].copy()
    out[prefix + "action"] = t.data["action"].copy()
    out[prefix + "reward"] = t.data["reward"].copy()
    out[prefix + "nonterminal"] = t.data["nonterminal"].astype(np.uint8)
    out[prefix + "meta"] = np.array([t.index, int(t.full), mem.t, t.size], dtype=np.int64)
    out[prefix + "max"] = np.float32(t.max)


def gen_replay():
    """ReplayMemory.append / sample / update_priorities / iterator on small rings."""
    out = {}
    cases = []
    for name, cap, n, B, fill, beta in (("c64n3", 64, 3, 8, 100, 0.4), ("c64n1", 64, 1, 8, 40, 0.7),
                                        ("c128n20", 128, 20, 4, 300, 1.0), ("c500n3", 500, 3, 32, 700, 0.4),
                                        ("c128n36", 128, 36, 4, 300, 0.5)):   # history + n = 40 > 32 window records
        rs = np.random.RandomState(11)
        np.random.seed(5)
        mem = ref_memory.ReplayMemory(make_args(multi_step=n, priority_weight=beta), cap)
        ep_len = 0
        for i in range(fill):
            terminal = bool(rs.uniform() < 0.08) or ep_len > 30
            ep_len = 0 if terminal else ep_len + 1
            mem.append(pattern_state(i), int(rs.randint(0, 6)), float(rs.randint(-1, 2)), terminal)
        # spread priorities (the reference only ever writes them through update_priorities)
        ts = mem.transitions.tree_start
        count = cap if mem.transitions.full else mem.transitions.index
        mem.update_priorities(np.arange(count) + ts, rs.uniform(0.01, 4, count).astype(np.float32))
        pfx = name + "_"
        dump_ring(mem, out, pfx)
        n_samples = 6
        attempts = []
        for s in range(n_samples):
            with UniformRecorder() as rec:
                tidx, states, actions, returns, nstates, nonterm, weights = mem.sample(B)
            u = np.stack(rec.calls)  # [attempts, B]
            attempts.append(u.shape[0])
            out[f"{pfx}s{s}_u01"] = u
            out[f"{pfx}s{s}_tidx"] = np.asarray(tidx, np.int64)
            out[f"{pfx}s{s}_states"] = states.numpy()
            out[f"{pfx}s{s}_actions"] = actions.numpy()
            out[f"{pfx}s{s}_returns"] = returns.numpy()
            out[f"{pfx}s{s}_nstates"] = nstates.numpy()
            out[f"{pfx}s{s}_nonterm"] = nonterm.numpy()
            out[f"{pfx}s{s}_weights"] = weights.numpy()
            # write back priorities like agent.py:100 does, so later samples see an updated tree
            raw = rs.uniform(0, 2, B).astype(np.float32)
            mem.update_priorities(tidx, raw)
            out[f"{pfx}s{s}_raw"] = raw
            out[f"{pfx}s{s}_tree_after"] = mem.transitions.sum_tree.copy()
            out[f"{pfx}s{s}_max_after"] = np.float32(mem.transitions.max)
        # validation iterator (memory.py:162-180): first 12 states
        it = iter(mem)
        out[pfx + "iter"] = np.stack([next(it).numpy() for _ in range(12)])
        cases.append(dict(name=name, cap=cap, n=n, B=B, fill=fill, beta=beta, attempts=attempts))
    np.savez_compressed(os.path.join(OUT, "replay.npz"), **out)
    return cases


def history_case_frame(i):
    """uint8 frame the reference stores for pattern_state(i) (memory.py:106); tests regenerate it with the same two lines."""
    return pattern_state(i)[-1].mul(255).to(torch.uint8).numpy().reshape(-1)


def as_frame_bytes(x, what):
    """float32 gathered frames -> uint8, asserting that every value is byte / 255 (0 for a blank)."""
    u8 = np.rint(x * 255).astype(np.uint8)
    assert np.array_equal(u8.astype(np.float32) / np.float32(255), x), what
    return u8


def gen_replay_history():
    """ReplayMemory.append / sample / the iterator at histories other than 4, on rings of short episodes (terminal
    probability 0.3) so that most windows cross an episode boundary.  Gathered frames are stored as their bytes; the ring's
    frames are history_case_frame(i) of the i-th append and are not stored."""
    out = {}
    cases = []
    for name, H, n, cap, B, fill in (("h1n3", 1, 3, 64, 8, 90), ("h2n1", 2, 1, 64, 8, 90), ("h5n5", 5, 5, 64, 6, 100),
                                     ("h5n2", 5, 2, 64, 6, 40), ("h8n3", 8, 3, 64, 4, 100),
                                     ("h16n48", 16, 48, 128, 2, 150)):   # history + n = 64: the longest window
        rs = np.random.RandomState(23)
        np.random.seed(29)
        mem = ref_memory.ReplayMemory(make_args(history_length=H, multi_step=n), cap)
        for i in range(fill):
            mem.append(pattern_state(i), int(rs.randint(0, 6)), float(rs.randint(-1, 2)), bool(rs.uniform() < 0.3))
        ts = mem.transitions.tree_start
        count = cap if mem.transitions.full else mem.transitions.index
        mem.update_priorities(np.arange(count) + ts, rs.uniform(0.01, 4, count).astype(np.float32))
        pfx = name + "_"
        ring = {}
        dump_ring(mem, ring, pfx)
        frames = ring.pop(pfx + "frames")
        expect = np.zeros_like(frames)
        for i in range(fill):
            expect[i % cap] = history_case_frame(i)
        assert np.array_equal(frames, expect), "ring frames are history_case_frame of each append"
        out.update(ring)
        attempts = []
        for s in range(2):
            with UniformRecorder() as rec:
                tidx, states, actions, returns, nstates, nonterm, weights = mem.sample(B)
            attempts.append(len(rec.calls))
            out[f"{pfx}s{s}_u01"] = np.stack(rec.calls)
            out[f"{pfx}s{s}_tidx"] = np.asarray(tidx, np.int64)
            out[f"{pfx}s{s}_states"] = as_frame_bytes(states.numpy(), "states")
            out[f"{pfx}s{s}_nstates"] = as_frame_bytes(nstates.numpy(), "next states")
            out[f"{pfx}s{s}_actions"] = actions.numpy()
            out[f"{pfx}s{s}_returns"] = returns.numpy()
            out[f"{pfx}s{s}_nonterm"] = nonterm.numpy()
            mem.update_priorities(tidx, rs.uniform(0, 2, B).astype(np.float32))
            out[f"{pfx}s{s}_tree_after"] = mem.transitions.sum_tree.copy()
        # the iterator (memory.py:162-180) at both ends of the ring and in between, through its own current_idx
        cur = np.array(sorted({0, 1, H - 1, cap // 2, cap - H + 1, cap - 1} - {cap}), np.int64)
        it = iter(mem)
        iters = []
        for c in cur:
            it.current_idx = int(c)
            iters.append(as_frame_bytes(next(it).numpy(), "iterator state"))
        out[pfx + "iter_cur"] = cur
        out[pfx + "iter"] = np.stack(iters)
        cases.append(dict(name=name, history=H, n=n, cap=cap, B=B, fill=fill, attempts=attempts))
    np.savez_compressed(os.path.join(OUT, "replay_history.npz"), **out)
    return cases


def gen_append():
    """Step-by-step append on a tiny ring, incl. wrap-around and the running max (memory.py:105-108, 56-61)."""
    out = {}
    rs = np.random.RandomState(3)
    mem = ref_memory.ReplayMemory(make_args(), 8)
    steps = 19
    states = []
    for i in range(steps):
        st = torch.from_numpy(rs.uniform(0, 1, (4, 84, 84)).astype(np.float32))
        if i == 4:
            st[-1, 0, :8] = torch.tensor([0.0, 1.0, 0.5, 1 / 255, 2 / 255, 254 / 255, 0.999999, 0.00392])
        a, r, term = int(rs.randint(0, 6)), float(rs.randint(-1, 2)), bool(i in (5, 6, 13))
        mem.append(st, a, r, term)
        if i == 9:  # raise the running max through an update, later appends must use it
            mem.update_priorities(np.array([mem.transitions.tree_start + 2]), np.array([9.0], np.float32))
        states.append(st[-1].numpy())
        out[f"a{i}_args"] = np.array([a, r, int(term)], np.float64)
        out[f"a{i}_tree"] = mem.transitions.sum_tree.copy()
        out[f"a{i}_meta"] = np.array([mem.transitions.index, int(mem.transitions.full), mem.t], np.int64)
        out[f"a{i}_max"] = np.float32(mem.transitions.max)
    out["last_frames_f32"] = np.stack(states)
    dump_ring(mem, out, "final_")
    np.savez_compressed(os.path.join(OUT, "append.npz"), **out)


def gen_pow():
    rs = np.random.RandomState(9)
    x = np.concatenate([rs.uniform(0, 5, 4000), rs.uniform(0, 1e-3, 1000), [0.0, 1.0, 4.0, 1e-30]]).astype(np.float32)
    out = {"x": x}
    for om in (0.5, 0.6, 1.0, 0.25):
        out[f"pow_{om}"] = np.power(x, om)
    np.savez_compressed(os.path.join(OUT, "pow.npz"), **out)


# --------------------------------------------------------------------------------------------
class StubNet(torch.nn.Module):
    """Stands in for DQN inside the unmodified Agent.learn: returns (log_)softmax over atoms of fixed
    logit tensors, exactly the tail of model.py:76-79, so that gradients w.r.t. the logits are observable."""

    def __init__(self, q_for_states, q_for_next, states, next_states):
        super().__init__()
        self.q_s = torch.nn.Parameter(q_for_states.clone())
        self.q_ns = torch.nn.Parameter(q_for_next.clone())
        self._s, self._ns = states, next_states

    def forward(self, x, log=False):
        q = self.q_s if x is self._s else self.q_ns
        assert x is self._s or x is self._ns
        return torch.nn.functional.log_softmax(q, dim=2) if log else torch.nn.functional.softmax(q, dim=2)

    def reset_noise(self):
        pass


class SpyStates(torch.Tensor):
    """states tensor whose new_zeros() result (the `m` buffer of agent.py:89) is remembered."""
    made = []

    def new_zeros(self, *a, **k):
        t = torch.zeros(*a)
        SpyStates.made.append(t)
        return t


class FakeMem:
    def __init__(self, batch):
        self.batch = batch
        self.got = None

    def sample(self, B):
        return self.batch

    def update_priorities(self, idxs, pri):
        self.got = (idxs, np.array(pri, copy=True))


def gen_learn():
    """agent.py:61-100 run unmodified on stub nets: loss, m, grad w.r.t. pre-softmax logits."""
    out = {}
    cases = []
    for name, B, A, n, seed, atoms in (("b32a6", 32, 6, 3, 0, 51), ("b1a3", 1, 3, 1, 1, 51), ("b64a18", 64, 18, 20, 2, 51),
                                       ("b8a4sharp", 8, 4, 3, 3, 51), ("b8a4z101", 8, 4, 3, 4, 101)):   # 101 atoms: > 64
        g = torch.Generator().manual_seed(seed)
        rs = np.random.RandomState(seed)
        args = make_args(batch_size=B, multi_step=n, norm_clip=1e9, atoms=atoms)
        ag = ref_agent.Agent(make_args(batch_size=B, multi_step=n, norm_clip=1e9, architecture="data-efficient",
                                       hidden_size=8, atoms=atoms), FakeEnv(A))
        Z = args.atoms
        scale = 6.0 if "sharp" in name else 1.5
        q_s = torch.randn(B, A, Z, generator=g) * scale
        q_ns = torch.randn(B, A, Z, generator=g) * scale
        q_t = torch.randn(B, A, Z, generator=g) * scale
        states = torch.zeros(B, 1).as_subclass(SpyStates)
        nstates = torch.zeros(B, 1)
        actions = torch.from_numpy(rs.randint(0, A, B).astype(np.int64))
        gam = np.array([args.discount ** i for i in range(n)], np.float32)
        rew = rs.randint(-1, 2, (B, n)).astype(np.float32)
        returns = torch.from_numpy(rew) @ torch.from_numpy(gam)
        ret_np = returns.numpy().copy()
        if B >= 8:  # clamp cases and exact-integer b cases
            ret_np[0], ret_np[1], ret_np[2], ret_np[3] = 12.0, -12.0, 0.0, 10.0
            returns = torch.from_numpy(ret_np)
        nonterm = torch.from_numpy((rs.uniform(size=(B, 1)) > 0.3).astype(np.float32))
        w = rs.uniform(0.2, 1.0, B).astype(np.float32)
        w /= w.max()
        weights = torch.from_numpy(w)
        idxs = np.arange(B, dtype=np.int64)
        ag.online_net = StubNet(q_s, q_ns, states, nstates)
        ag.target_net = StubNet(q_t, q_t, None, nstates)
        ag.target_net._s = object()
        ag.optimiser = torch.optim.SGD(ag.online_net.parameters(), lr=0.0)
        mem = FakeMem((idxs, states, actions, returns, nstates, nonterm, weights))
        SpyStates.made.clear()
        ag.learn(mem)
        m = SpyStates.made[-1]
        assert ag.online_net.q_ns.grad is None
        p = name + "_"
        out[p + "q_s"], out[p + "q_ns"], out[p + "q_t"] = q_s.numpy(), q_ns.numpy(), q_t.numpy()
        out[p + "actions"], out[p + "returns"], out[p + "nonterm"] = actions.numpy(), returns.numpy(), nonterm.numpy()
        out[p + "weights"] = weights.numpy()
        out[p + "support"] = ag.support.numpy()
        out[p + "loss"] = mem.got[1]
        out[p + "m"] = m.numpy().copy()
        out[p + "grad"] = ag.online_net.q_s.grad.numpy().copy()
        with torch.no_grad():
            pns = torch.softmax(q_ns, 2)
            out[p + "astar"] = (ag.support.expand_as(pns) * pns).sum(2).argmax(1).numpy()
        cases.append(dict(name=name, B=B, A=A, n=n, Z=Z, V_min=args.V_min, V_max=args.V_max,
                          discount=args.discount, delta_z=ag.delta_z))
    np.savez_compressed(os.path.join(OUT, "learn.npz"), **out)
    return cases


# --------------------------------------------------------------------------------------------
def gen_noise():
    """NoisyLinear.reset_noise (model.py:32-40) with the torch.randn draws recorded."""
    out = {}
    torch.manual_seed(0)
    orig = torch.randn
    for name, fin, fout in (("l37x19", 37, 19), ("l576x64", 576, 64), ("l512x51", 512, 51)):
        layer = ref_model.NoisyLinear(fin, fout, std_init=0.1)
        rec = []

        def wrapped(*a, **k):
            x = orig(*a, **k)
            rec.append(x.clone())
            return x

        torch.randn = wrapped
        try:
            layer.reset_noise()
        finally:
            torch.randn = orig
        assert len(rec) == 2 and rec[0].numel() == fin and rec[1].numel() == fout  # eps_in drawn first
        out[name + "_x_in"], out[name + "_x_out"] = rec[0].numpy(), rec[1].numpy()
        out[name + "_w_eps"] = layer.weight_epsilon.numpy().copy()
        out[name + "_b_eps"] = layer.bias_epsilon.numpy().copy()
    np.savez_compressed(os.path.join(OUT, "noise.npz"), **out)


def gen_model_step():
    """One full unmodified Agent.learn on a tiny data-efficient DQN: parameters before/after, gradients, loss.
    Used by the end-to-end learner test (GPU path vs reference CPU path, float tolerance)."""
    out = {}
    torch.manual_seed(1)
    np.random.seed(1)
    B, A = 4, 3
    args = make_args(batch_size=B, architecture="data-efficient", hidden_size=64, multi_step=3)
    ag = ref_agent.Agent(args, FakeEnv(A))
    for k, v in ag.online_net.state_dict().items():
        out["sd0." + k] = v.numpy().copy()
    rs = np.random.RandomState(4)
    states = torch.from_numpy(rs.randint(0, 256, (B, 4, 84, 84)).astype(np.float32)) / 255
    nstates = torch.from_numpy(rs.randint(0, 256, (B, 4, 84, 84)).astype(np.float32)) / 255
    actions = torch.from_numpy(rs.randint(0, A, B).astype(np.int64))
    returns = torch.tensor([0.0, 1.0, -1.99, 2.9701])
    nonterm = torch.tensor([[1.0], [1.0], [0.0], [1.0]])
    weights = torch.tensor([1.0, 0.5, 0.7, 0.9])
    mem = FakeMem((np.arange(B), states, actions, returns, nstates, nonterm, weights))
    # record the target net's noise draw (agent.py:74)
    rec = []
    orig = torch.randn

    def wrapped(*a, **k):
        x = orig(*a, **k)
        rec.append(x.clone())
        return x

    torch.randn = wrapped
    try:
        ag.learn(mem)
    finally:
        torch.randn = orig
    assert len(rec) == 8
    for i, x in enumerate(rec):
        out[f"target_randn{i}"] = x.numpy()
    for k, v in ag.target_net.state_dict().items():
        if "epsilon" in k:
            out["target_eps." + k] = v.numpy().copy()
    out["states_u8"] = (states * 255).round().to(torch.uint8).numpy()
    out["nstates_u8"] = (nstates * 255).round().to(torch.uint8).numpy()
    out["actions"], out["returns"], out["nonterm"], out["weights"] = actions.numpy(), returns.numpy(), nonterm.numpy(), weights.numpy()
    out["loss"] = mem.got[1]
    for k, p in ag.online_net.named_parameters():
        out["grad." + k] = p.grad.numpy().copy()
    for k, v in ag.online_net.state_dict().items():
        out["sd1." + k] = v.numpy().copy()
    np.savez_compressed(os.path.join(OUT, "model_step.npz"), **out)


# --------------------------------------------------------------------------------------------
def sample_stride(numel):
    """Sub-sampling rule of the full-update fixtures (tests/helpers.py holds the same function): small tensors are
    kept whole, large ones every stride-th element (odd strides, so every row and column is hit)."""
    return 1 if numel <= 4096 else (5 if numel <= 40000 else (23 if numel <= 200000 else 199))


class RandnRecorder:
    """Records every torch.randn draw (model.py:33) made while active."""

    def __init__(self):
        self.calls = []
        self.orig = torch.randn

    def __enter__(self):
        def wrapped(*a, **k):
            x = self.orig(*a, **k)
            self.calls.append(x.clone())
            return x

        torch.randn = wrapped
        return self

    def __exit__(self, *a):
        torch.randn = self.orig

    def split(self):
        """reset order is eps_in then eps_out per layer (model.py:37-38): returns (all eps_in draws, all eps_out draws)."""
        assert len(self.calls) == 8
        return torch.cat(self.calls[0::2]).numpy(), torch.cat(self.calls[1::2]).numpy()


def gen_full_update(name, arch, hidden, n, cap, B, A, steps, seed):
    """`steps` consecutive UNMODIFIED `dqn.reset_noise(); dqn.learn(mem)` pairs (main.py:150-151) at a benchmarked network
    shape on a small real ReplayMemory: recorded noise draws, sampled indices, per-sample losses, gradients, parameters and
    the sum tree after every step.  Initial parameters and frames are regenerated by the test from the seeds (checked by
    SHA); large tensors are sub-sampled (sample_stride) and additionally pinned by float64 sums."""
    out = {}
    torch.manual_seed(seed)
    np.random.seed(seed + 100)
    args = make_args(batch_size=B, multi_step=n, architecture=arch, hidden_size=hidden)
    ag = ref_agent.Agent(args, FakeEnv(A))
    sd0 = torch.cat([p.detach().reshape(-1) for _, p in ag.online_net.named_parameters()])
    mem = ref_memory.ReplayMemory(args, cap)
    rs = np.random.RandomState(seed + 7)
    fill = cap + cap // 3
    frames = rs.randint(0, 256, (fill, 84, 84), dtype=np.uint8)     # the test re-draws exactly this
    ep = 0
    for i in range(fill):
        st = torch.zeros(4, 84, 84)
        st[-1] = (torch.from_numpy(frames[i]).float() + 0.5) / 255     # mul(255) + truncation gives back frames[i]
        terminal = bool(rs.uniform() < 0.03) or ep > 60
        ep = 0 if terminal else ep + 1
        mem.append(st, int(rs.randint(0, A)), float(rs.randint(-1, 2)), terminal)
    ts = mem.transitions.tree_start
    mem.update_priorities(np.arange(cap) + ts, rs.uniform(0.01, 4, cap).astype(np.float32))
    ring = np.zeros((cap, 84, 84), np.uint8)
    for i in range(fill):
        ring[i % cap] = frames[i]
    assert np.array_equal(mem.transitions.data["state"], ring)
    t = mem.transitions
    out["ring_sum_tree"], out["ring_timestep"], out["ring_action"] = t.sum_tree.copy(), t.data["timestep"].copy(), t.data["action"].copy()
    out["ring_reward"], out["ring_nonterminal"] = t.data["reward"].copy(), t.data["nonterminal"].astype(np.uint8)
    out["ring_meta"] = np.array([t.index, int(t.full), mem.t, t.size], dtype=np.int64)
    out["ring_max"] = np.float32(t.max)
    strides = {k: sample_stride(p.numel()) for k, p in ag.online_net.named_parameters()}
    attempts = []
    for k in range(steps):
        with RandnRecorder() as rec:
            ag.reset_noise()                                            # main.py:150
        out[f"s{k}_online_x_in"], out[f"s{k}_online_x_out"] = rec.split()
        got = {}
        orig_update = mem.update_priorities

        def spy(idxs, pri):
            got["idxs"], got["loss"] = np.array(idxs, copy=True), np.array(pri, copy=True)
            return orig_update(idxs, pri)

        mem.update_priorities = spy
        try:
            with RandnRecorder() as rec, UniformRecorder() as urec:
                ag.learn(mem)                                           # main.py:151
        finally:
            del mem.update_priorities
        out[f"s{k}_target_x_in"], out[f"s{k}_target_x_out"] = rec.split()
        attempts.append(len(urec.calls))
        out[f"s{k}_tidx"], out[f"s{k}_loss"] = got["idxs"].astype(np.int64), got["loss"].astype(np.float32)
        for key, p in ag.online_net.named_parameters():
            for kind, v in (("grad", p.grad), ("param", p.detach())):
                flat = v.reshape(-1)
                out[f"s{k}_{kind}.{key}"] = flat[::strides[key]].numpy().copy()
                out[f"s{k}_{kind}sum.{key}"] = np.array([float(flat.double().sum()), float((flat.double() ** 2).sum())])
        out[f"s{k}_tree_after"] = t.sum_tree.copy()
        out[f"s{k}_max_after"] = np.float32(t.max)
    np.savez_compressed(os.path.join(OUT, f"update_{name}.npz"), **out)
    return dict(name=name, arch=arch, hidden=hidden, n=n, cap=cap, B=B, A=A, steps=steps, seed=seed, fill=fill,
                attempts=attempts, sd0_sha=sha(sd0.numpy()), frames_sha=sha(ring), strides=strides)


def gen_ref_pickle():
    """A replay file written by the UNMODIFIED reference exactly like main.py:94-100 does (bz2 + pickle of the whole
    ReplayMemory object), plus the arrays it holds, for the load-a-reference-file test (SURVEY 8(f).3)."""
    import bz2
    import pickle
    rs = np.random.RandomState(21)
    mem = ref_memory.ReplayMemory(make_args(multi_step=3), 64)
    for i in range(83):
        mem.append(pattern_state(i), int(rs.randint(0, 6)), float(rs.randint(-1, 2)), bool(i in (6, 15, 40, 41)))
    mem.update_priorities(np.arange(64) + mem.transitions.tree_start, rs.uniform(0.1, 3, 64).astype(np.float32))
    with bz2.open(os.path.join(OUT, "ref_memory.pkl.bz2"), "wb") as f:
        pickle.dump(mem, f)
    out = {}
    dump_ring(mem, out, "")
    np.random.seed(3)
    with UniformRecorder() as rec:
        tidx, states, actions, returns, nstates, nonterm, weights = mem.sample(4)
    out["u01"], out["tidx"], out["states"], out["returns"] = np.stack(rec.calls), np.asarray(tidx, np.int64), states.numpy(), returns.numpy()
    out["weights"] = weights.numpy()
    np.savez_compressed(os.path.join(OUT, "ref_memory.npz"), **out)


def gen_ref_pickle_state():
    """The state the reference's memory.py holds after loading save_reference_pickle()'s file of the ref_memory.npz arrays
    (export direction of SURVEY 8(f).3), checked here to sample like the original object did."""
    import subprocess
    import tempfile
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
    sys.path.insert(0, os.path.dirname(HERE))
    from helpers import golden, loaded_reference_state, write_reference_pickle_of_golden
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "mem.pkl")
        write_reference_pickle_of_golden(path)
        state = loaded_reference_state(path, REF)
        code = (f"import sys, pickle, numpy as np; sys.path.insert(0, {REF!r}); import memory\n"
                f"mem = pickle.load(open({path!r}, 'rb'))\nnp.random.seed(3)\n"
                "print(' '.join(str(int(i)) for i in mem.sample(4)[0]))\n")
        res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True)
    assert [int(x) for x in res.stdout.split()] == golden("ref_memory")["tidx"].tolist()
    with open(os.path.join(OUT, "ref_pickle_state.json"), "w") as f:
        json.dump(state, f, indent=1, sort_keys=True)


def main():
    os.makedirs(OUT, exist_ok=True)
    manifest = dict(reference="Kaixhin/Rainbow@1745b184c3dfc03d4ffa3ce2342ced9996b39a60", numpy=np.__version__,
                    torch=torch.__version__, python=sys.version.split()[0])
    manifest["big_trees"] = gen_tree()
    manifest["replay_cases"] = gen_replay()
    manifest["replay_history_cases"] = gen_replay_history()
    gen_append()
    gen_pow()
    manifest["learn_cases"] = gen_learn()
    gen_noise()
    gen_model_step()
    # whole-update trajectories at the benchmarked shapes: C2 (canonical / 512, n 3) and C3 (data-efficient / 256, n 20)
    manifest["update_cases"] = [gen_full_update("c2", "canonical", 512, 3, 512, 32, 6, 3, 11),
                                gen_full_update("c3", "data-efficient", 256, 20, 2048, 32, 6, 3, 12)]
    gen_ref_pickle()
    gen_ref_pickle_state()
    with open(os.path.join(OUT, "MANIFEST.json"), "w") as f:
        json.dump(manifest, f, indent=1)
    for fn in sorted(os.listdir(OUT)):
        print(fn, os.path.getsize(os.path.join(OUT, fn)))


def main_replay_history():
    """Only tests/golden/replay_history.npz and its MANIFEST.json key; every other fixture is left as it is."""
    path = os.path.join(OUT, "MANIFEST.json")
    with open(path) as f:
        manifest = json.load(f)
    manifest["replay_history_cases"] = gen_replay_history()
    with open(path, "w") as f:
        json.dump(manifest, f, indent=1)
    print("replay_history.npz", os.path.getsize(os.path.join(OUT, "replay_history.npz")))


if __name__ == "__main__":
    if sys.argv[1:] == ["ref_pickle_state"]:
        gen_ref_pickle_state()
    elif sys.argv[1:] == ["replay_history"]:
        main_replay_history()
    else:
        main()
