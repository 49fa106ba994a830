"""numpy reference of the dormant-neuron statistics and of ReDo recycling (rb_neuron_scores, rb_redo_mask,
rb_redo_recycle): score sums and normalised scores in float64, the mask with the kernel's threshold arithmetic (float64, the
layer mean summed in neuron order), and the rewritten flat parameter and moment buffers with theta0 drawn by
reset_ref's bit formula on the stream word "REDO"."""
import numpy as np

import philox_ref as P
import reset_ref as R

REDO_STREAM = 0x5245444F   # "REDO"
CHUNK = 64                 # addends of one fp32 partial sum of rb_neuron_scores
SUM_REL_BOUND = (CHUNK - 1) * 2.0 ** -24   # |kernel sum - exact| <= this x exact, for non-negative activations


def score_sums(act):
    """Sum over rows and positions of act [R, C, ...] per neuron, in float64 (exact to 2^-53 relative per addition)."""
    a = np.asarray(act, dtype=np.float64)
    return a.reshape(a.shape[0], a.shape[1], -1).sum(axis=(0, 2))


def normalised_scores(sums, count):
    """s_i / mean_j s_j of one layer (inf / nan where the mean is 0), s_i = sums_i / count."""
    s = np.asarray(sums, np.float64) / np.float64(count)
    with np.errstate(divide="ignore", invalid="ignore"):
        return s / (np.cumsum(s)[-1] / np.float64(s.size))


def mask_ref(sums, layers, tau):
    """rb_redo_mask: layers [(offset, neurons, count)]; returns (mask uint8 over all neurons, [dormant count per layer]).
    np.cumsum adds in index order, as thread 0 of the layer's CTA does."""
    sums = np.asarray(sums, np.float64)
    mask = np.zeros(sums.size, np.uint8)
    counts = []
    for off, n, count in layers:
        s = sums[off:off + n] / np.float64(count)
        threshold = np.float64(np.float32(tau)) * (np.cumsum(s)[-1] / np.float64(n))
        d = s <= threshold
        mask[off:off + n] = d
        counts.append(int(d.sum()))
    return mask, counts


def draw_words(seed, pass_index, idx):
    """reset_ref.draw_words with the fourth counter word REDO_STREAM."""
    idx = np.asarray(idx, dtype=np.int64)
    q = (idx >> 2).astype(np.uint64)
    k = int(pass_index)
    ctr = np.stack([np.full(q.shape, k & 0xFFFFFFFF, np.uint64), np.full(q.shape, (k >> 32) & 0xFFFFFFFF, np.uint64),
                    q & np.uint64(0xFFFFFFFF), np.full(q.shape, REDO_STREAM, np.uint64)], axis=-1).astype(np.uint32)
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], dtype=np.uint32)
    return P.philox4x32_10(ctr, key)[np.arange(idx.size), idx & 3]


def theta0(seed, pass_index, idx, bound, constant):
    w = draw_words(seed, pass_index, idx)
    u = (w >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)
    r = np.float32(2.0) * u - np.float32(1.0)
    return R.fma32(np.full(r.size, bound, np.float32), r, np.full(r.size, constant, np.float32))


def incoming_indices(block, neurons):
    """Flat indices of an incoming block (offset, elements per neuron, ...) for one neuron or an array of neurons."""
    off, per, *_ = block
    i = np.atleast_1d(np.asarray(neurons, dtype=np.int64))
    return (off + i[:, None] * per + np.arange(per, dtype=np.int64)).ravel()


def outgoing_indices(block, neurons):
    """Flat indices of an outgoing block (offset, rows, row stride, elements per neuron) for one or several neurons."""
    off, rows, stride, span = block
    i = np.atleast_1d(np.asarray(neurons, dtype=np.int64))
    return (off + np.arange(rows, dtype=np.int64)[None, :, None] * stride + i[:, None, None] * span +
            np.arange(span, dtype=np.int64)).ravel()


def recycle_ref(param, exp_avg, exp_avg_sq, table, mask, seed, pass_index):
    """rb_redo_recycle on host copies.  `table`: rainbow_b200.agent.redo_table's rows.  Incoming elements of every dormant
    neuron are re-drawn first, then the outgoing elements of every dormant neuron are zeroed (an element that is both
    ends up +0); the moments of both become 0.  Returns (param, exp_avg, exp_avg_sq, written bool mask)."""
    p, m, v = (np.array(x, dtype=np.float32, copy=True) for x in (param, exp_avg, exp_avg_sq))
    written = np.zeros(p.size, bool)
    dormant = [np.flatnonzero(mask[row["mask_offset"]:row["mask_offset"] + row["neurons"]]) for row in table]
    for row, d in zip(table, dormant):
        for blk in row["incoming"] if d.size else ():
            idx = incoming_indices(blk, d)
            p[idx] = theta0(seed, pass_index, idx, blk[4], blk[5])
            written[idx] = True
    for row, d in zip(table, dormant):
        for blk in row["outgoing"] if d.size else ():
            idx = outgoing_indices(blk, d)
            p[idx] = 0.0
            written[idx] = True
    m[written] = 0.0
    v[written] = 0.0
    return p, m, v, written
