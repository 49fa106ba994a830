"""numpy statement of ReplayMemory.extend (rb_append_bulk, DESIGN §23): k records appended at once leave the ring as k
appends in order would.

- timesteps: t_j = t0 + j before the first nonzero flag, else j - r_j - 1, r_j the last index < j whose flag is nonzero
  (terminal or final observation); the episode counter carried past the block follows all k flags;
- records: only the last min(k, size) survive, record j at slot (head + j) mod size;
- tree: every touched leaf gets the running max (0 for a final observation), then every ancestor of a touched leaf is
  recomputed level by level as fl32(left + right).  A missing right child (odd sizes, which only the oracle builds) reads 0.
"""
import numpy as np

FINAL = 2


def timesteps(flags, t0):
    """(t [k] int64, the episode counter after the block) by an exclusive max-scan of the reset positions."""
    flags = np.asarray(flags)
    k = flags.size
    j = np.arange(k, dtype=np.int64)
    marks = np.where(flags != 0, j, -1)
    incl = np.maximum.accumulate(marks) if k else marks
    r = np.concatenate([[-1], incl[:-1]]) if k else marks
    t = np.where(r < 0, int(t0) + j, j - r - 1)
    t_end = int(t0) + k if (k == 0 or incl[-1] < 0) else int(k - 1 - incl[-1])
    return t, t_end


def tree_start(size):
    return 2 ** (int(size) - 1).bit_length() - 1


def rebuild(tree, size, slots, values):
    """Leaves at `slots` set to `values`, then their ancestors recomputed level by level in float32.  Returns a new tree."""
    ts = tree_start(size)
    out = np.concatenate([np.asarray(tree, np.float32), np.zeros(1, np.float32)])   # index len(tree) reads 0
    nodes = np.asarray(slots, np.int64) + ts
    out[nodes] = np.asarray(values, np.float32)
    nodes = np.unique(nodes)
    while nodes.size and nodes[0] != 0:
        nodes = np.unique((nodes - 1) // 2)
        out[nodes] = out[2 * nodes + 1] + out[2 * nodes + 2]   # float32 + float32, round to nearest
    return out[:-1]


def extend(ring, actions, rewards, flags, frames=None):
    """ring: dict(size, tree, timestep, action, reward, nonterminal, index, full, t, max[, frames]) -> the same dict after
    the k records (frames [k, ...] optional).  `max` is the running max, which appends leave unchanged."""
    size, head, k = int(ring["size"]), int(ring["index"]), len(flags)
    flags = np.asarray(flags, np.uint8)
    t, t_end = timesteps(flags, ring["t"])
    out = {key: (v.copy() if isinstance(v, np.ndarray) else v) for key, v in ring.items()}
    first = max(0, k - size)
    j = np.arange(first, k)
    slots = (head + j) % size
    fin = flags[j] == FINAL
    out["timestep"][slots] = t[j].astype(np.int32)
    out["action"][slots] = np.where(fin, 0, np.asarray(actions, np.int32)[j])
    out["reward"][slots] = np.where(fin, np.float32(0), np.asarray(rewards, np.float32)[j])
    out["nonterminal"][slots] = np.where(fin, FINAL, np.where(flags[j] != 0, 0, 1)).astype(np.uint8)
    if frames is not None:
        out["frames"][slots] = np.asarray(frames)[j].reshape(len(j), -1)
    leaves = np.where(fin, np.float32(0), np.float32(ring["max"])).astype(np.float32)
    out["tree"] = rebuild(ring["tree"], size, slots, leaves)
    out["index"] = (head + k) % size
    out["full"] = bool(ring["full"]) or head + k >= size
    out["t"] = t_end
    return out
