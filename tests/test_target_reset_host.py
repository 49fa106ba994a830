"""Polyak target updates and shrink-and-perturb resets without a GPU: every refusal of rb_target_ema and rb_param_reset
(answered before any launch), the Agent's option checks, the checkpoint's new scalar checks, the exact-fma and theta0
references of tests/reset_ref.py, and the reset table's bounds against torch's own initialisation rules."""
import argparse
import ctypes as C
import math

import numpy as np
import pytest
import torch

import philox_ref as P
import reset_ref as R

RB_ERR_INVAL, RB_ERR_RANGE = -22, -34
ONE = 4096   # a pointer that is never dereferenced: validation fails first


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


def net_args(arch):
    return argparse.Namespace(atoms=51, hidden_size=512 if arch == "canonical" else 256, architecture=arch,
                              history_length=4, noisy_std=0.1)


# ---- rb_target_ema -------------------------------------------------------------------------------------------------------
def test_target_ema_refusals_without_gpu():
    L = lib()
    # target, param, n, tau, gate, stream
    assert L.rb_target_ema(None, ONE, 8, 0.5, None, None) == RB_ERR_INVAL
    assert b"null" in L.rb_last_error()
    assert L.rb_target_ema(ONE, None, 8, 0.5, None, None) == RB_ERR_INVAL
    assert L.rb_target_ema(ONE, 1 << 20, -1, 0.5, None, None) == RB_ERR_INVAL
    for tau in (0.0, -0.0, -0.5, 1.0000001, 2.0, float("nan"), float("inf"), -float("inf")):
        assert L.rb_target_ema(ONE, 1 << 20, 8, tau, None, None) == RB_ERR_RANGE, tau
        assert b"tau" in L.rb_last_error()
    # overlapping buffers: the same buffer, one inside the other, a partial overlap either way
    for t, p, n in ((ONE, ONE, 8), (ONE, ONE + 4, 8), (ONE + 28, ONE, 8), (ONE, ONE + 4 * 7, 8)):
        assert L.rb_target_ema(t, p, n, 0.5, None, None) == RB_ERR_INVAL, (t, p, n)
        assert b"overlap" in L.rb_last_error()
    # n == 0 launches nothing (so it answers without a GPU as well)
    assert L.rb_target_ema(ONE, ONE + 64, 0, 0.5, None, None) == 0


# ---- rb_param_reset ------------------------------------------------------------------------------------------------------
def segments(*rows):
    from rainbow_b200 import _lib
    return (_lib.ResetSegment * max(1, len(rows)))(*[_lib.ResetSegment(*r) for r in rows])


def test_param_reset_refusals_without_gpu():
    L = lib()
    good = [(0, 100, 0.1, 0.0, 0.5), (128, 64, 0.0, 0.05, 0.0), (192, 8, 0.2, 0.0, 1.0)]

    def call(rows, n=256, n_segs=None, param=ONE):
        s = segments(*rows)
        return L.rb_param_reset(param, n, s, len(rows) if n_segs is None else n_segs, 7, 0, None)

    assert L.rb_param_reset(None, 256, segments(*good), 3, 7, 0, None) == RB_ERR_INVAL
    assert L.rb_param_reset(ONE, 256, None, 3, 7, 0, None) == RB_ERR_INVAL
    assert b"null" in L.rb_last_error()
    for k in (0, -1, 33):
        assert call(good, n_segs=k) == RB_ERR_RANGE, k
    too_many = [(4 * i, 2, 0.1, 0.0, 0.5) for i in range(33)]
    assert call(too_many) == RB_ERR_RANGE
    bad_segments = [
        [(-4, 8, 0.1, 0.0, 0.5)],                                  # before 0
        [(250, 8, 0.1, 0.0, 0.5)],                                 # past n
        [(0, 257, 0.1, 0.0, 0.5)],                                 # longer than n
        [(0, 0, 0.1, 0.0, 0.5)],                                   # empty
        [(0, -3, 0.1, 0.0, 0.5)],
        [(128, 8, 0.1, 0.0, 0.5), (0, 8, 0.1, 0.0, 0.5)],          # unsorted
        [(0, 100, 0.1, 0.0, 0.5), (99, 8, 0.1, 0.0, 0.5)],         # overlapping
        [(0, 100, 0.1, 0.0, 0.5), (0, 100, 0.1, 0.0, 0.5)],        # the same segment twice
    ]
    for rows in bad_segments:
        assert call(rows) == RB_ERR_RANGE, rows
        assert b"segment" in L.rb_last_error()
    for b in (-0.1, float("nan"), float("inf")):
        assert call([(0, 8, b, 0.0, 0.5)]) == RB_ERR_RANGE, b
        assert call([(0, 8, 0.0, b, 0.5)]) == RB_ERR_RANGE, b
    for a in (-0.01, 1.01, float("nan"), float("inf")):
        assert call([(0, 8, 0.1, 0.0, a)]) == RB_ERR_RANGE, a
        assert b"alpha" in L.rb_last_error()
    assert call(good, n=-1) == RB_ERR_RANGE                       # no segment fits a negative n
    # one bad row anywhere refuses the whole call
    assert call(good + [(200, 8, 0.1, 0.0, 1.5)]) == RB_ERR_RANGE


def test_signatures_kernel_ids_and_segment_layout():
    from rainbow_b200 import _lib
    assert len(_lib.SIGNATURES["rb_target_ema"][1]) == 6 and len(_lib.SIGNATURES["rb_param_reset"][1]) == 7
    assert _lib.ALL_KERNEL_IDS[-2:] == ["target_ema", "param_reset"]
    assert _lib.ALL_KERNEL_IDS[:len(_lib.PROFILE_IDS)] == _lib.PROFILE_IDS
    # rb_reset_segment: int64 offset, count; float bound, constant, alpha (32 bytes with the trailing padding)
    assert C.sizeof(_lib.ResetSegment) == 32 and _lib.ResetSegment.bound.offset == 16 and _lib.ResetSegment.alpha.offset == 24


def test_kernel_ids_are_the_header_enum():
    """_lib.ALL_KERNEL_IDS against the RB_K_* enum itself: every name, in enum order, RB_KERNEL_COUNT of them; and the
    library answers rb_profile_collect for the last id and refuses the count."""
    import os
    import re

    from rainbow_b200 import _lib
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include",
                               "rainbow_b200.h")).read()
    body = re.search(r"enum\s*\{([^}]*RB_KERNEL_COUNT[^}]*)\}", header).group(1)
    names = [n.strip().split("=")[0].strip() for n in body.split(",") if n.strip()]
    assert names[-1] == "RB_KERNEL_COUNT" and "= 0" in body.split(",")[0]
    assert [n[len("RB_K_"):].lower() for n in names[:-1]] == _lib.ALL_KERNEL_IDS
    tot, n = C.c_double(), C.c_int()
    L = lib()
    assert L.rb_profile_collect(len(_lib.ALL_KERNEL_IDS) - 1, C.byref(tot), C.byref(n)) == 0 and n.value == 0
    assert L.rb_profile_collect(len(_lib.ALL_KERNEL_IDS), C.byref(tot), C.byref(n)) == RB_ERR_INVAL


# ---- Agent options and checkpoint scalars ---------------------------------------------------------------------------------
def test_agent_option_checks():
    from rainbow_b200.agent import target_reset_options
    ns = argparse.Namespace
    assert target_reset_options(ns()) == (0.0, 0, (1.0, 0.0))
    assert target_reset_options(ns(target_tau=None, reset_interval=None, reset_shrink_encoder=None)) == (0.0, 0, (1.0, 0.0))
    assert target_reset_options(ns(target_tau=0.005, reset_interval=4, reset_shrink_encoder=0.5, reset_shrink_head=0.2)) == \
        (0.005, 4, (0.5, 0.2))
    assert target_reset_options(ns(target_tau=1, reset_shrink_encoder=0.0, reset_shrink_head=1.0)) == (1.0, 0, (0.0, 1.0))
    assert target_reset_options(ns(target_tau=1e-44))[0] == 1e-44       # a subnormal fp32: the kernel takes it
    for bad in (dict(target_tau=-0.1), dict(target_tau=1.5), dict(target_tau=float("nan")), dict(target_tau=1e-46),
                dict(target_tau=1.0 + 1e-9), dict(reset_interval=-1),
                dict(reset_interval=2.5), dict(reset_interval=True), dict(reset_shrink_encoder=1.1),
                dict(reset_shrink_encoder=-0.5), dict(reset_shrink_head=float("nan")), dict(reset_shrink_head=2.0)):
        with pytest.raises(ValueError):
            target_reset_options(ns(**bad))


def test_checkpoint_scalar_checks():
    from rainbow_b200 import _lib
    from rainbow_b200.checkpoint import _SCALARS, check_reset_scalars
    seed, count = _SCALARS[("learner", "reset_seed")], _SCALARS[("learner", "reset_count")]
    assert seed(None, None) and count(None, None), "absent = a manifest from before the keys existed"
    assert seed(0, None) and seed(2 ** 63 - 1, None) and count(0, None) and count(12, None)
    for v in (-1, 2 ** 63, True, 1.5, "3"):
        assert not seed(v, None), v
    for v in (-1, 2 ** 63, False, 2.0):
        assert not count(v, None), v
    check_reset_scalars(dict(reset_seed=5, reset_count=0))
    check_reset_scalars(dict(learn_calls=3))
    for half in (dict(reset_seed=5), dict(reset_count=2), dict(reset_seed=None, reset_count=1)):
        with pytest.raises(_lib.RainbowB200Error, match="together"):
            check_reset_scalars(half)


# ---- references ----------------------------------------------------------------------------------------------------------
def test_fma32_is_the_correctly_rounded_fused_multiply_add():
    from fractions import Fraction
    rs = np.random.RandomState(3)
    a = rs.uniform(-2, 2, 4000).astype(np.float32)
    b = rs.uniform(-2, 2, 4000).astype(np.float32)
    c = (rs.uniform(-1, 1, 4000) * 10.0 ** rs.randint(-9, 3, 4000)).astype(np.float32)
    # cases near ties: c = -fl32(a b) leaves only the rounding error of a b, and c = half an ulp of a b
    c[:500] = -(a[:500] * b[:500])
    ab = (a[500:1000].astype(np.float64) * b[500:1000]).astype(np.float32)
    c[500:1000] = (np.spacing(ab) / 2).astype(np.float32)
    got = R.fma32(a, b, c)

    def exact(x, y, z):
        v = Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))
        lo = np.float32(float(v))                        # float() rounds the rational correctly to float64 ...
        # ... and from there to float32 may double-round: settle it on the rational value
        cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        errs = [abs(Fraction(float(q)) - v) for q in cands]
        best = min(errs)
        ties = [q for q, e in zip(cands, errs) if e == best]
        return ties[0] if len(ties) == 1 else [q for q in ties if (int(np.float32(q).view(np.uint32)) & 1) == 0][0]

    want = np.array([exact(x, y, z) for x, y, z in zip(a, b, c)], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_ema_reference():
    rs = np.random.RandomState(4)
    t, p = rs.randn(1000).astype(np.float32), rs.randn(1000).astype(np.float32)
    assert np.array_equal(R.ema_ref(t, p, 1.0), p), "tau = 1 copies"
    for tau in (1e-3, 0.005, 0.5):
        got = R.ema_ref(t, p, tau)
        keep = np.float32(1) - np.float32(tau)
        assert np.abs(got.astype(np.float64) - (np.float64(np.float32(tau)) * p + np.float64(keep * t))).max() <= \
            np.abs(got).max() * 2.0 ** -23
        assert not np.array_equal(got, t) and not np.array_equal(got, p)


def test_theta0_reference_bit_formula():
    seed, k = 0x0123456789ABCDEF, (3 << 32) + 5
    idx = np.arange(1000, 1040, dtype=np.int64)
    w = R.draw_words(seed, k, idx)
    for j in (1000, 1001, 1003, 1037):
        word = P.philox4x32_10(np.array([5, 3, j >> 2, R.RESET_STREAM], np.uint32),
                               np.array([0x89ABCDEF, 0x01234567], np.uint32))[j & 3]
        assert w[j - 1000] == word
        u = float(word >> 8) * 2.0 ** -24
        assert R.theta0(seed, k, np.array([j]), 0.25, 0.0)[0] == np.float32(0.25 * (2 * u - 1))   # exact: one rounding
        assert R.theta0(seed, k, np.array([j]), 0.0, 0.0375)[0] == np.float32(0.0375)
    th = R.theta0(seed, k, np.arange(200000), 0.1, 0.0)
    assert th.min() >= np.float32(-0.1) and th.max() < np.float32(0.1)
    assert abs(th.mean()) < 1e-3 and abs(th.std() - 0.1 / math.sqrt(3)) < 1e-3
    assert not np.array_equal(th[:1000], R.theta0(seed, k + 1, np.arange(1000), 0.1, 0.0)), "the reset index is in the counter"
    assert not np.array_equal(th[:1000], R.theta0(seed + 1, k, np.arange(1000), 0.1, 0.0)), "the seed is the key"


def test_reset_reference_blend():
    rs = np.random.RandomState(5)
    param = rs.randn(512).astype(np.float32)
    segs = [(0, 100, 0.1, 0.0, 1.0), (128, 64, 0.0, 0.05, 0.0), (256, 77, 0.3, 0.0, 0.5)]
    out, drawn = R.reset_ref(param, segs, 11, 2)
    assert np.array_equal(out[:100], param[:100]), "alpha = 1 is a no-op"
    assert (out[128:192] == np.float32(0.05)).all(), "alpha = 0 re-draws (a constant here)"
    assert np.array_equal(out[256:333], R.fma32(np.full(77, 0.5, np.float32), param[256:333], np.float32(0.5) * drawn[2]))
    outside = np.ones(512, bool)
    for off, n, *_ in segs:
        outside[off:off + n] = False
    assert np.array_equal(out[outside], param[outside])


# ---- the reset table against torch's own initialisation ----------------------------------------------------------------
@pytest.mark.parametrize("arch,n_tensors", [("canonical", 22), ("data-efficient", 20)])
def test_reset_table_bounds_are_torchs(arch, n_tensors):
    from torch import nn

    from rainbow_b200.agent import ENCODER, HEAD, FusedClipAdam, reset_table
    from rainbow_b200.model import DQN, NoisyLinear
    torch.manual_seed(0)
    net = DQN(net_args(arch), 6)
    opt = FusedClipAdam(net, lr=1e-4, eps=1e-4, max_norm=10.0)
    table = reset_table(net, opt.offsets)
    assert len(table) == n_tensors <= 32
    named = list(net.named_parameters())
    end = 0
    for (name, p), (off, count, bound, constant, group), o in zip(named, table, opt.offsets):
        assert off == o and count == p.numel() and off >= end
        end = off + count
        owner, kind = name.rsplit(".", 1)
        m = net.get_submodule(owner)
        if isinstance(m, nn.Conv2d):
            assert group == ENCODER and constant == 0.0
            # torch's rules: kaiming_uniform_(a=sqrt(5)) for the weight, 1 / sqrt(fan_in) for the bias
            fan_in, _ = nn.init._calculate_fan_in_and_fan_out(m.weight)
            gain = nn.init.calculate_gain("leaky_relu", math.sqrt(5))
            torch_bound = math.sqrt(3.0) * gain / math.sqrt(fan_in) if kind == "weight" else 1.0 / math.sqrt(fan_in)
            assert math.isclose(bound, torch_bound, rel_tol=1e-12) and np.float32(bound) == np.float32(torch_bound), name
            fresh = nn.Conv2d(m.in_channels, m.out_channels, m.kernel_size, stride=m.stride)
            w = getattr(fresh, kind).detach().abs()
            assert float(w.max()) <= np.float32(bound) and float(w.max()) > 0.9 * bound, name
        else:
            assert isinstance(m, NoisyLinear) and group == HEAD
            fresh = NoisyLinear(m.in_features, m.out_features, std_init=m.std_init)
            v = getattr(fresh, kind).detach()
            if kind.endswith("_sigma"):       # NoisyLinear.reset_parameters fills a constant: the table's, in fp32
                assert bound == 0.0 and (v == torch.tensor(np.float32(constant))).all(), name
            else:                             # uniform_(-b, b) with b = 1 / sqrt(in_features)
                assert constant == 0.0 and math.isclose(bound, 1.0 / math.sqrt(fan_in_of(fresh)), rel_tol=1e-15)
                assert float(v.abs().max()) <= np.float32(bound) and float(v.abs().max()) > 0.9 * bound, name
    assert end <= opt.numel
    assert sum(count for _, count, *_ in table) == sum(p.numel() for _, p in named) < opt.numel, "padding is left out"


def fan_in_of(linear):
    """torch's fan-in rule for a [out, in] weight."""
    from torch import nn
    return nn.init._calculate_fan_in_and_fan_out(linear.weight_mu)[0]
