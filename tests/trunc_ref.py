"""The truncation-aware n-step gather (rb_gather_trunc) stated in plain numpy, record by record.

A final-observation record F (nonterminal byte FINAL, ReplayMemory.append_truncated) holds the observation a time limit
stopped its episode at.  For a sample at record idx let k be the offset of the first F among records idx + 1 .. idx + n - 1,
or n if there is none.  The sample is gathered over a window of k steps: states from records idx - h + 1 .. idx, next
states from idx + k - h + 1 .. idx + k, both blanked backwards from their newest frame at an episode start (timestep 0)
exactly like the fixed-horizon gather; the return sums the k rewards idx .. idx + k - 1 with gamma_pow[j], each zero once
an episode started after idx; the nonterminal is fl32(nt * gamma_k) with nt the stored byte of idx + k read as 0 / 1 (0
when an episode started in between) and gamma_k = gamma_pow[k] for k < n, gamma_n for k = n: the discount form a loss
launched with gamma_n = 1 reads.

Written apart from oracle/rb_oracle.c on purpose: tests/test_truncation_host.py checks this statement against the
oracle's fixed-horizon gather at n = k, which is what makes it a reference for the kernels."""
import numpy as np

FINAL = 2


def cut(tree, idx, n):
    """k for the sample at data index idx (see the module docstring)."""
    rec = (int(idx) + 1 + np.arange(n - 1)) % tree.size
    hits = np.flatnonzero(tree.nonterminal[rec] == FINAL)
    return int(hits[0]) + 1 if hits.size else n


def gather_trunc(tree, didx, history, n, gamma_pow, gamma_n):
    """(states, actions, returns, next_states, nonterminals [B, 1], k per sample) of rb_gather_trunc for a row of n,
    gamma_pow (at least n entries) and gamma_n."""
    didx = np.asarray(didx, np.int64)
    B, size = didx.size, tree.size
    gp = np.asarray(gamma_pow, np.float32)
    states = np.empty((B, history, 84, 84), np.float32)
    nstates = np.empty((B, history, 84, 84), np.float32)
    actions = np.empty(B, np.int64)
    returns = np.empty(B, np.float32)
    nonterm = np.empty((B, 1), np.float32)
    ks = np.empty(B, np.int64)
    for b, idx in enumerate(didx):
        k = cut(tree, idx, n)
        ks[b] = k
        rec = (idx - (history - 1) + np.arange(history + k)) % size
        first = tree.timestep[rec] == 0

        def blank(s):
            if s < history - 1:
                return bool(first[s + 1:history].any())
            if s >= history:
                return bool(first[history:s + 1].any())
            return False

        frames = [np.zeros(84 * 84, np.float32) if blank(s) else tree.frames[rec[s]].astype(np.float32) / np.float32(255)
                  for s in range(history + k)]
        states[b] = np.stack(frames[:history]).reshape(history, 84, 84)
        nstates[b] = np.stack(frames[k:k + history]).reshape(history, 84, 84)
        actions[b] = tree.action[idx % size]
        acc = np.float32(0)
        for j in range(k):
            r = np.float32(0) if blank(history - 1 + j) else tree.reward[(idx + j) % size]
            acc = np.float32(acc + np.float32(r * gp[j]))
        returns[b] = acc
        nt = np.float32(0) if blank(history - 1 + k) or tree.nonterminal[(idx + k) % size] == 0 else np.float32(1)
        gamma_k = gp[k] if k < n else np.float32(gamma_n)
        nonterm[b, 0] = np.float32(nt * gamma_k)
    return states, actions, returns, nstates, nonterm, ks


def final_ring(tree, idxs, ks):
    """Writes a final-observation record k records after each idx of the host OracleTree `tree` (in order) as
    ReplayMemory.append_truncated leaves one: records idx .. idx + k - 1 nonterminal transitions of one episode, F
    continuing it with action 0 and reward 0, and the records after F renumbered from an episode start up to the next
    start already there."""
    size = tree.size
    for idx, k in zip(idxs, ks):
        for j in range(1, int(k) + 1):   # idx .. F one episode
            cur = (int(idx) + j) % size
            tree.nonterminal[(cur - 1) % size] = 1
            tree.timestep[cur] = tree.timestep[(cur - 1) % size] + 1
        f = (int(idx) + int(k)) % size
        tree.nonterminal[f], tree.action[f], tree.reward[f] = FINAL, 0, np.float32(0)
        j, t = (f + 1) % size, 0
        while tree.timestep[j] != 0 or t == 0:
            tree.timestep[j] = t
            j, t = (j + 1) % size, t + 1
    return tree
