"""numpy / float64 reference of the noisy nets' device noise (rb_noise_factors, rb_noisy_resample, rb_noisy_outer).

Normal g of stream `which` (0 = eps_in, 1 = eps_out) for draw `counter` of a net with key `seed`, as normal4 in
rainbow_b200/csrc/rb_internal.cuh forms it: Philox4x32-10 with counter (c_lo, c_hi, g >> 2, 0x4E4F4953 + which) and key
(seed_lo, seed_hi); words (x, y) give normals 4k, 4k + 1 as (r cos, r sin) of box_muller, words (z, w) normals 4k + 2, 4k + 3.
The layer sits in the normal's index: the streams of a net are the layers' eps_in (eps_out) back to back in noisy_layers()
order.  The Box-Muller here runs in float64 on the device's exact uniforms (philox_ref.box_muller_uniforms), so it differs
from the device only by the device's logf / sqrtf / sincospif and its rounded products: |x_dev - x| <= TAU_X max(r, 1)
(tests/test_noise_host.py derives TAU_X and holds it to the house rule).

Factors f(x) = sign(x) sqrt|x| (model.py's scale_noise) in float64; the device's fp32 factor of its own normal is within
factor_bound(x, r) of it.  From given fp32 normals the device's factors are scale(x) bitwise (sqrt is correctly rounded),
and weight_epsilon is outer(f_out, f_in), fl32 products, bitwise."""
import numpy as np

import philox_ref as P

NOISE_STREAM = 0x4E4F4953        # "NOIS": + 0 for eps_in, + 1 for eps_out
U63 = 2 ** 63 - 1
TAU_X = 2e-6                     # |x_dev - x| <= TAU_X max(r, 1), r the float64 Box-Muller radius
TAIL = float(np.sqrt(-2.0 * np.log(2.0 ** -32)))   # 6.6604: the largest radius, at u1 = 2^-32


def words(seed, counter, which, n):
    """uint32 [ceil(n / 4)][4]: the Philox words of normals 0 .. n - 1 of stream `which`."""
    blk = np.arange(-(-n // 4), dtype=np.uint64)
    full = lambda v: np.full(blk.size, v, np.uint64)
    ctr = np.stack([full(counter & 0xFFFFFFFF), full((counter >> 32) & 0xFFFFFFFF), blk, full(NOISE_STREAM + which)],
                   axis=-1).astype(np.uint32)
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], dtype=np.uint32)
    return P.philox4x32_10(ctr, key)


def box_muller(a, b):
    """float64 (r cos(2 pi u2), r sin(2 pi u2), r) of box_muller's words a, b, r = sqrt(-2 ln u1)."""
    u1, u2 = P.box_muller_uniforms(a, b)
    r = np.sqrt(-2.0 * np.log(u1))
    t = np.pi * (2.0 * u2)
    return r * np.cos(t), r * np.sin(t), r


def normals(seed, counter, which, n, radius=False):
    """float64 [n]: normals 0 .. n - 1 of stream `which` for draw `counter`; radius=True also returns each one's r."""
    w = words(seed, counter, which, n)
    x0, x1, r0 = box_muller(w[:, 0], w[:, 1])
    x2, x3, r1 = box_muller(w[:, 2], w[:, 3])
    x = np.stack([x0, x1, x2, x3], axis=-1).reshape(-1)[:n]
    if not radius:
        return x
    return x, np.stack([r0, r0, r1, r1], axis=-1).reshape(-1)[:n]


def f64(x):
    """f(x) = sign(x) sqrt|x| in float64."""
    return np.sign(x) * np.sqrt(np.abs(x))


def scale(x):
    """scale_noise of fp32 normals, bitwise: fl32(sign(x) sqrt_rn(|x|)), +0 at x = +-0."""
    x = np.asarray(x, np.float32)
    s = np.where(x > 0, np.float32(1), np.where(x < 0, np.float32(-1), np.float32(0))).astype(np.float32)
    return (s * np.sqrt(np.abs(x))).astype(np.float32)


def outer(f_out, f_in):
    """weight_epsilon [out][in]: fl32(f_out[o] f_in[i]) (__fmul_rn), bitwise."""
    return np.multiply.outer(np.asarray(f_out, np.float32), np.asarray(f_in, np.float32)).astype(np.float32)


def draw(seed, counter, n_in, n_out):
    """One draw of a net whose layers hold n_in / n_out factors in all: float64 (x_in, r_in, x_out, r_out)."""
    return normals(seed, counter, 0, n_in, radius=True) + normals(seed, counter, 1, n_out, radius=True)


def factors(seed, counter, in_features, out_features):
    """[(f_in, f_out)] in float64 per layer, the layers in noisy_layers() order, for draw `counter` of key `seed`."""
    x_in, _, x_out, _ = draw(seed, counter, sum(in_features), sum(out_features))
    oi, oo = np.cumsum([0] + list(in_features)), np.cumsum([0] + list(out_features))
    return [(f64(x_in[oi[l]:oi[l + 1]]), f64(x_out[oo[l]:oo[l + 1]])) for l in range(len(in_features))]


def factor_bound(x, r):
    """Bound on |f_dev - f(x)| for the device's fp32 factor of its own normal of x (float64 x and r):
    delta = TAU_X max(r, 1) bounds |x_dev - x|.  f is not Lipschitz at 0, so: where |x| > delta the signs agree and
    |sqrt|x_dev| - sqrt|x|| <= delta / sqrt|x| (< sqrt(delta)); where |x| <= delta the sign may flip, and
    sqrt|x_dev| + sqrt|x| <= sqrt(2 delta) covers both cases.  Plus sqrt_rn's half ulp, 2^-24 sqrt|x_dev| <=
    2^-24 (sqrt|x| + sqrt(delta))."""
    x, r = np.abs(np.asarray(x, np.float64)), np.asarray(r, np.float64)
    delta = TAU_X * np.maximum(r, 1.0)
    near = x <= delta
    main = np.where(near, np.sqrt(2.0 * delta), delta / np.sqrt(np.where(near, 1.0, x)))
    return main + 2.0 ** -24 * (np.sqrt(x) + np.sqrt(delta))


def factor_check(f_dev, x, r):
    """(largest |f_dev - f(x)| / factor_bound, number of sign flips where |x| > delta) for fp32 device factors."""
    f_dev = np.asarray(f_dev, np.float64)
    ratio = np.abs(f_dev - f64(x)) / factor_bound(x, r)
    flips = (np.sign(f_dev) != np.sign(x)) & (np.abs(x) > TAU_X * np.maximum(r, 1.0))
    return float(ratio.max(initial=0.0)), int(flips.sum())


def agent_seeds(initial_seed, rank):
    """(online, target) noise seeds of an Agent built after torch's seed `initial_seed`, on data-parallel rank `rank`:
    DQN takes initial_seed & (2^63 - 1), and the Agent makes the two nets and the ranks distinct."""
    s = int(initial_seed) & U63
    return (s * 2 + 1 + 7919 * rank) & U63, (s * 2 + 2 + 7919 * rank) & U63
