"""numpy references of the Polyak target update (rb_target_ema) and of the shrink-and-perturb reset (rb_param_reset): an
exact fp32 fused multiply-add, the blend t <- fma(tau, p, fl32(1 - tau) t), and theta0 drawn from Philox4x32-10 with the
bit formula of include/rainbow_b200.h."""
import numpy as np

import philox_ref as P

RESET_STREAM = 0x52534554   # "RSET"


def fma32(a, b, c):
    """fl32(a * b + c) with a single rounding, for fp32 arrays a, b, c.  a * b is exact in float64 (24 x 24 bits); the sum
    is taken exactly as s + e (TwoSum) and rounded to odd in float64 -- 53 >= 24 + 2 bits, so the final rounding to fp32
    gives the correctly rounded fma (no double rounding)."""
    a, b, c = (np.asarray(x, dtype=np.float32).astype(np.float64) for x in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)                          # exact: p + c = s + e
    odd = np.ascontiguousarray(s).view(np.uint64) & np.uint64(1)
    fix = (e != 0) & (odd == 0)
    s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def ema_ref(target, param, tau):
    """rb_target_ema: fma(tau, p, fl32(fl32(1 - tau) * t)), every operation in fp32."""
    tau = np.float32(tau)
    keep = np.float32(np.float32(1.0) - tau)
    t = np.asarray(target, dtype=np.float32)
    return fma32(np.full_like(t, tau), param, keep * t)


def draw_words(seed, reset_index, idx):
    """The Philox word of every flat index in `idx`: word (j & 3) of Philox4x32-10 with key `seed` and counter
    (k_lo, k_hi, j >> 2, RESET_STREAM)."""
    idx = np.asarray(idx, dtype=np.int64)
    q = (idx >> 2).astype(np.uint64)
    k = int(reset_index)
    ctr = np.stack([np.full(q.shape, k & 0xFFFFFFFF, np.uint64), np.full(q.shape, (k >> 32) & 0xFFFFFFFF, np.uint64),
                    q & np.uint64(0xFFFFFFFF), np.full(q.shape, RESET_STREAM, np.uint64)], axis=-1).astype(np.uint32)
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], dtype=np.uint32)
    words = P.philox4x32_10(ctr, key)
    return words[np.arange(idx.size), idx & 3]


def theta0(seed, reset_index, idx, bound, constant):
    """fma(bound, r, constant), r = 2u - 1, u = (w >> 8) 2^-24 (r is exact in fp32)."""
    w = draw_words(seed, reset_index, idx)
    u = (w >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)
    r = np.float32(2.0) * u - np.float32(1.0)
    n = r.size
    return fma32(np.full(n, bound, np.float32), r, np.full(n, constant, np.float32))


def reset_ref(param, segments, seed, reset_index):
    """rb_param_reset on a host copy: segments [(offset, count, bound, constant, alpha)]; returns (new param, theta0 of every
    segment)."""
    out = np.array(param, dtype=np.float32, copy=True)
    drawn = []
    for off, count, bound, constant, alpha in segments:
        idx = np.arange(off, off + count, dtype=np.int64)
        th0 = theta0(seed, reset_index, idx, bound, constant)
        a = np.float32(alpha)
        keep = np.float32(np.float32(1.0) - a)
        out[off:off + count] = fma32(np.full(count, a, np.float32), out[off:off + count], keep * th0)
        drawn.append(th0)
    return out, drawn
