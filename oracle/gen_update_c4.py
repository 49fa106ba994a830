#!/usr/bin/env python
"""Whole-update fixture at C4's learner shape from the UNMODIFIED reference: canonical / 512, n 3, 6 actions, batch 512.

    python oracle/gen_update_c4.py        # writes tests/golden/update_c4.npz only

Three `dqn.reset_noise(); dqn.learn(mem)` pairs (main.py:150-151) on a 16384-transition ReplayMemory, driven like
oracle/gen_golden.py::gen_full_update (same fill, same recorders), stored compactly and self-described (the case metadata
is inside the file, tests/golden/MANIFEST.json is not involved):
  * the noise draws as the torch CPU generator state right after the Agent is built: every later torch.randn of the
    reference is a reset_noise draw (checked here), so the test regenerates them from that state;
  * sum trees as their leaves (the reference's nodes are the float32 sums of their children, checked here) and, after each
    step, as the SHA-256 of the whole tree plus the sampled leaves;
  * at most 256 evenly strided elements of every gradient / parameter tensor per step, plus float64 sums of each.
16384 transitions keep every stratified segment (32 leaves) wide next to the invalid window around the write head, so the
reference's redraw loop (memory.py:127-132) ends quickly.  At this batch size one of the reference's draws retrieves a leaf
twice in about one step in three (seeds 13-15 each have such a step); seed 16's three batches are free of that, which the
per-leaf check of the written priorities needs."""
import hashlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import gen_golden as G  # noqa: E402  (puts the reference on sys.path)

CASE = dict(name="c4", arch="canonical", hidden=512, n=3, cap=16384, B=512, A=6, steps=3, seed=16)
SAMPLES = 256


def sample_stride(numel):
    """Stride of the per-tensor samples (tests/test_gpu_head_large_f64.py holds the same rule)."""
    return -(-numel // SAMPLES)


def tree_from_leaves(leaves, tree_start):
    """The reference's sum tree: leaves after tree_start, every node the float32 sum of its two children."""
    tree = np.zeros(tree_start + leaves.size, np.float32)
    tree[tree_start:] = leaves
    lo = tree_start
    while lo > 0:
        plo = (lo - 1) // 2
        par = np.arange(plo, lo)
        tree[par] = tree[2 * par + 1] + tree[2 * par + 2]
        lo = plo
    return tree


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    c = CASE
    out = {}
    torch.manual_seed(c["seed"])
    np.random.seed(c["seed"] + 100)
    args = G.make_args(batch_size=c["B"], multi_step=c["n"], architecture=c["arch"], hidden_size=c["hidden"])
    ag = G.ref_agent.Agent(args, G.FakeEnv(c["A"]))
    rng_after_init = torch.get_rng_state()
    sd0 = torch.cat([p.detach().reshape(-1) for _, p in ag.online_net.named_parameters()])
    mem = G.ref_memory.ReplayMemory(args, c["cap"])
    rs = np.random.RandomState(c["seed"] + 7)
    cap, fill = c["cap"], c["cap"] + c["cap"] // 3
    frames = rs.randint(0, 256, (fill, 84, 84), dtype=np.uint8)           # tests/helpers.py::update_case_ring re-draws this
    ep = 0
    for i in range(fill):
        st = torch.zeros(4, 84, 84)
        st[-1] = (torch.from_numpy(frames[i]).float() + 0.5) / 255
        terminal = bool(rs.uniform() < 0.03) or ep > 60
        ep = 0 if terminal else ep + 1
        mem.append(st, int(rs.randint(0, c["A"])), float(rs.randint(-1, 2)), terminal)
    t = mem.transitions
    mem.update_priorities(np.arange(cap) + t.tree_start, rs.uniform(0.01, 4, cap).astype(np.float32))
    ring = np.zeros((cap, 84, 84), np.uint8)
    for i in range(fill):
        ring[i % cap] = frames[i]
    assert np.array_equal(t.data["state"], ring)
    assert np.array_equal(tree_from_leaves(t.sum_tree[t.tree_start:], t.tree_start), t.sum_tree)
    out["ring_leaves"], out["ring_timestep"], out["ring_action"] = t.sum_tree[t.tree_start:].copy(), t.data["timestep"].copy(), t.data["action"].copy()
    out["ring_reward"], out["ring_nonterminal"] = t.data["reward"].copy(), t.data["nonterminal"].astype(np.uint8)
    out["ring_meta"] = np.array([t.index, int(t.full), mem.t, t.size], dtype=np.int64)
    out["ring_max"] = np.float32(t.max)
    names = [k for k, _ in ag.online_net.named_parameters()]
    strides = {k: sample_stride(p.numel()) for k, p in ag.online_net.named_parameters()}
    draws, attempts = [], []
    for k in range(c["steps"]):
        with G.RandnRecorder() as rec:
            ag.reset_noise()                                              # main.py:150
        draws += rec.calls
        got = {}
        orig_update = mem.update_priorities

        def spy(idxs, pri):
            got["idxs"], got["loss"] = np.array(idxs, copy=True), np.array(pri, copy=True)
            return orig_update(idxs, pri)

        mem.update_priorities = spy
        try:
            with G.RandnRecorder() as rec, G.UniformRecorder() as urec:
                ag.learn(mem)                                             # main.py:151
        finally:
            del mem.update_priorities
        assert len(rec.calls) == 8
        draws += rec.calls
        attempts.append(len(urec.calls))
        out[f"s{k}_tidx"], out[f"s{k}_loss"] = got["idxs"].astype(np.int64), got["loss"].astype(np.float32)
        assert len(set(got["idxs"].tolist())) == c["B"], "a leaf drawn twice in one batch: pick another seed"
        for key, p in ag.online_net.named_parameters():
            for kind, v in (("grad", p.grad), ("param", p.detach())):
                flat = v.reshape(-1)
                out[f"s{k}_{kind}.{key}"] = flat[::strides[key]].numpy().copy()
                out[f"s{k}_{kind}sum.{key}"] = np.array([float(flat.double().sum()), float((flat.double() ** 2).sum())])
        out[f"s{k}_tree_sha"] = np.array(sha(t.sum_tree))
        out[f"s{k}_tree_leaves"] = t.sum_tree[got["idxs"]].copy()
        out[f"s{k}_max_after"] = np.float32(t.max)
    # every torch.randn after the Agent was built is a noise draw: the test regenerates them from this generator state
    torch.set_rng_state(rng_after_init)
    assert all(torch.equal(torch.randn(d.shape), d) for d in draws)
    out["rng_state"] = rng_after_init.numpy()
    out["draw_sizes"] = np.array([d.numel() for d in draws], np.int64)
    meta = dict(c, fill=fill, attempts=attempts, sd0_sha=sha(sd0.numpy()), frames_sha=sha(ring), tree_start=t.tree_start)
    for key, v in meta.items():
        out["case_" + key] = np.array(v)
    out["param_names"] = np.array(names)
    out["param_strides"] = np.array([strides[k] for k in names], np.int64)
    path = os.path.join(G.OUT, "update_c4.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes; attempts", attempts)


if __name__ == "__main__":
    main()
