"""CPU: the bounds tests/test_gpu_noise_f64.py holds the device noise to, and the reference of tests/noise_ref.py itself.

* TAU_X, the bound on |x_dev - x| / max(r, 1) for a device normal x_dev against the float64 Box-Muller x on the same
  uniforms.  The documented errors of the device's functions (CUDA C Programming Guide, Mathematical Functions, built
  without fast-math): logf 1 ulp, sqrtf 0 ulp (IEEE), sincospif 1 ulp each, products rounded to nearest (-2 logf and
  2 u2 exact).  An fp32 model of box_muller applies the two 1-ulp errors at their extreme (the correctly rounded result
  moved one more ulp, either way, so up to 1.5 ulp) on 2^21 pairs of words; TAU_X is at least 5x above its largest error
  and at least 5x below the largest error of each modelled slip on the same words: u1 without the + 1 (visible only where
  the word is small: fl32(a) + 1 == fl32(a) above 2^25), the pair's other element (r sin for r cos), and a neighbouring
  Philox word.
* factor_bound: f(x) = sign(x) sqrt|x| is not Lipschitz at 0; the bound derived from TAU_X holds for the model's factors
  and for normals placed at the extremes of TAU_X around 0, where a sign flip is accepted only for |x| <= delta.
* The reference against a standard normal at 2^22 draws per stream: a KS test, the radius never above
  sqrt(-2 ln 2^-32) = 6.6604 (u1 >= 2^-32, so no normal is larger), and no correlation between eps_in and eps_out,
  consecutive counters, or the online and target seeds.  With the GPU file holding the device to this reference per
  element, this is the statistical check of the device's draws.
* Pins: from injected normals the reference's factors and outer product equal oracle.noisy bitwise, and agent_seeds is
  the formula rainbow_b200/agent.py uses."""
import os
import re
import types

import numpy as np
import pytest
from scipy import stats

import noise_ref as N
import oracle
import philox_ref as P
from helpers import assert_bits_equal, golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAIRS = 2 ** 21
F32 = np.float32


def _pairs(seed=0x5EED, counter=3):
    w = N.words(seed, counter, 0, 2 * PAIRS)
    return np.concatenate([w[:, 0], w[:, 2]]), np.concatenate([w[:, 1], w[:, 3]]), w


def _ulp_away(v, s):
    """The fp32 value of v moved one ulp towards +inf (s > 0) or -inf (s < 0)."""
    v = np.asarray(v).astype(F32)
    return np.nextafter(v, F32(np.inf) if s > 0 else F32(-np.inf))


def fp32_model(a, b):
    """The device's box_muller in fp32 with logf and sincospif wrong by their documented ulp, every sign combination:
    [(x_cos, x_sin)] as float64 arrays, one pair per combination."""
    u1, u2 = P.box_muller_uniforms(a, b)
    L = np.log(u1)
    cos, sin = np.cos(np.pi * (2.0 * u2)), np.sin(np.pi * (2.0 * u2))
    out = []
    for s_log in (-1, 1):
        # logf(1) = 0 exactly (u1 = 1 where fl32(a) = 2^32): the model keeps ln u1 <= 0
        L_dev = np.minimum(_ulp_away(L, s_log).astype(np.float64), 0.0)
        r = np.sqrt(-2.0 * L_dev).astype(F32).astype(np.float64)   # sqrt_rn
        for s_trig in (-1, 1):
            # the exact product of two fp32 values is a float64: one rounding to fp32, as __fmul_rn
            out.append(tuple((r * _ulp_away(t, s_trig).astype(np.float64)).astype(F32).astype(np.float64) for t in (cos, sin)))
    return out


def _ratio(x, ref, r):
    e = np.abs(np.asarray(x, np.float64) - ref) / np.maximum(r, 1.0)
    return float(np.nan_to_num(e, nan=np.inf).max())


def test_tau_x_house_rule():
    a, b, w = _pairs()
    xc, xs, r = N.box_muller(a, b)
    model = max(max(_ratio(mc, xc, r), _ratio(ms, xs, r)) for mc, ms in fp32_model(a, b))
    _, u2 = P.box_muller_uniforms(a, b)
    with np.errstate(divide="ignore"):
        r_no1 = np.sqrt(-2.0 * np.log(a.astype(F32).astype(np.float64) * 2.0 ** -32))
    slips = {
        "u1 without + 1": _ratio(r_no1 * np.cos(np.pi * (2.0 * u2)), xc, r),
        "the pair's other element": _ratio(xs, xc, r),
        "a neighbouring Philox word": _ratio(N.box_muller(np.concatenate([w[:, 1], w[:, 3]]),
                                                          np.concatenate([w[:, 2], w[:, 0]]))[0], xc, r),
    }
    print(f"\nTAU_X {N.TAU_X:.2e}: model max {model:.3e} ({N.TAU_X / model:.1f}x below TAU_X); slips " +
          ", ".join(f"{k} {v:.3e} ({v / N.TAU_X:.1f}x)" for k, v in slips.items()))
    assert 1e-7 < model <= N.TAU_X / 5, "TAU_X at least 5x above the fp32 model's largest error"
    for k, v in slips.items():
        assert v >= 5 * N.TAU_X, f"TAU_X at least 5x below the slip '{k}' ({v:.3g})"
    # the + 1 matters only where fl32(a) + 1 != fl32(a): a < 2^25
    assert np.array_equal(r_no1[a >= 2 ** 25], r[a >= 2 ** 25])


def test_factor_bound_holds_for_the_model():
    a, b, _ = _pairs(seed=77, counter=2 ** 32 + 1)
    a, b = a[:PAIRS // 4], b[:PAIRS // 4]
    xc, xs, r = N.box_muller(a, b)
    worst = 0.0
    for mc, ms in fp32_model(a, b):
        for m, x in ((mc, xc), (ms, xs)):
            ratio, flips = N.factor_check(N.scale(m), x, r)
            assert flips == 0
            worst = max(worst, ratio)
    assert worst <= 1.0, worst
    # at the extremes of TAU_X around 0: x_dev = x +- delta, signs flip where |x| <= delta
    r = np.full(2001, 2.5)
    delta = N.TAU_X * 2.5
    x = np.linspace(-4 * delta, 4 * delta, 2001)
    for s in (-1.0, 1.0):
        x_dev = (x + s * delta).astype(F32)
        ratio, flips = N.factor_check(N.scale(x_dev), x, r)
        assert ratio <= 1.0 and flips == 0, (s, ratio, flips)
    # a bound that catches a real slip near zero: f of the other element's normal is far outside it
    assert N.factor_check(N.scale(xs.astype(F32)), xc, N.box_muller(a, b)[2])[0] > 100


def test_reference_is_a_standard_normal():
    n = 2 ** 22
    s_on, s_tg = N.agent_seeds(5, 0)
    x_in = N.normals(s_on, 9, 0, n)
    x_out = N.normals(s_on, 9, 1, n)
    x_next = N.normals(s_on, 10, 0, n)
    x_tg = N.normals(s_tg, 9, 0, n)
    for name, x in (("eps_in", x_in), ("eps_out", x_out)):
        ks = stats.kstest(x, "norm")
        assert ks.pvalue > 1e-3, (name, ks)
        assert abs(x.mean()) < 5 / np.sqrt(n) and abs(x.var() - 1.0) < 5 * np.sqrt(2.0 / n), name
    # the tail is cut where u1 = 2^-32: no normal beyond sqrt(-2 ln 2^-32)
    assert N.TAIL == pytest.approx(6.6604, abs=1e-4)
    _, r = N.normals(s_on, 9, 0, n, radius=True)
    assert np.isfinite(r).all() and r.max() <= N.TAIL and np.abs(x_in).max() <= N.TAIL
    assert N.box_muller(np.array([0], np.uint32), np.array([0], np.uint32))[2][0] == pytest.approx(N.TAIL, rel=1e-15)
    lim = 5 / np.sqrt(n)
    for what, y in (("eps_in / eps_out", x_out), ("consecutive counters", x_next), ("online / target seeds", x_tg)):
        assert abs(np.corrcoef(x_in, y)[0, 1]) < lim, what
        assert not np.array_equal(x_in[:64], y[:64]), what


def test_reference_layout():
    """Normal g of a stream does not depend on how many are drawn; layers are slices of the concatenated streams; the
    four normals of a Philox block are (r cos, r sin) of (x, y), then of (z, w); the two streams differ only in the
    fourth counter word."""
    seed, ctr = (2 ** 32 + 5), 2 ** 40 + 3
    full = N.normals(seed, ctr, 1, 4097)
    assert np.array_equal(N.normals(seed, ctr, 1, 7), full[:7])
    w = N.words(seed, ctr, 1, 8)
    c0, s0, _ = N.box_muller(w[1, 0], w[1, 1])
    c1, s1, _ = N.box_muller(w[1, 2], w[1, 3])
    assert np.array_equal(full[4:8], [c0, s0, c1, s1])
    ins, outs = (3136, 3136, 512, 512), (512, 512, 51, 306)
    fs = N.factors(seed, ctr, ins, outs)
    x_in, _, x_out, _ = N.draw(seed, ctr, sum(ins), sum(outs))
    assert np.array_equal(fs[2][0], N.f64(x_in[6272:6784])) and np.array_equal(fs[3][1], N.f64(x_out[1075:]))
    key = np.array([seed & 0xFFFFFFFF, seed >> 32], np.uint32)
    ctr_words = np.array([[ctr & 0xFFFFFFFF, ctr >> 32, 1, N.NOISE_STREAM + 1]], np.uint32)
    assert np.array_equal(P.philox4x32_10(ctr_words, key)[0], w[1])


def test_injected_normals_equal_the_oracle_bitwise():
    g = golden("noise")
    for name in ("l37x19", "l576x64", "l512x51"):
        x_in, x_out = g[name + "_x_in"], g[name + "_x_out"]
        w, b = oracle.noisy(x_in, x_out)
        assert_bits_equal(N.scale(x_out), b, f"{name}: bias_epsilon")
        assert_bits_equal(N.outer(N.scale(x_out), N.scale(x_in)), w, f"{name}: weight_epsilon")
    special = np.array([0.0, -0.0, 1e-45, -1e-45, 1.0, -4.0, 6.66], F32)
    assert_bits_equal(N.scale(special), np.array([0, 0, np.sqrt(F32(1e-45)), -np.sqrt(F32(1e-45)), 1, -2,
                                                  np.sqrt(F32(6.66))], F32), "scale_noise at the edges")


def test_agent_seeds_is_the_agents_formula():
    """agent_seeds against the two assignments in rainbow_b200/agent.py, evaluated on stand-in objects."""
    src = open(os.path.join(ROOT, "rainbow_b200", "agent.py")).read()
    exprs = {net: re.search(rf"^\s*self\.{net}\.noise_seed = (.+)$", src, re.M).group(1)
             for net in ("online_net", "target_net")}
    for s in (0, 1, 5, 2 ** 32 + 5, 2 ** 63 - 1, 2 ** 64 - 1):
        for rank in (0, 1, 7):
            base = s & N.U63                         # DQN: int(torch.initial_seed()) & (2^63 - 1)
            ns = types.SimpleNamespace(online_net=types.SimpleNamespace(noise_seed=base),
                                       target_net=types.SimpleNamespace(noise_seed=base), sync=types.SimpleNamespace(rank=rank))
            got = tuple(eval(exprs[n], {}, {"self": ns}) for n in ("online_net", "target_net"))
            assert got == N.agent_seeds(s, rank), (s, rank)
            assert got[0] != got[1] and all(0 <= v <= N.U63 for v in got)
    assert N.agent_seeds(5, 0) != N.agent_seeds(5, 1)
