"""Intensity augmentation and DrQ's K / M averaging without a GPU: the refusals of rb_gather_aug and
rb_c51_dueling_avg_loss_grad (answered before any launch), the replay's argument checks, the multiplier reference
(tests/drq_ref.py) and the tolerance of the averaged loss.

The tolerance is c51_ref.TAU, checked the way tests/test_c51_adam_bounds.py sizes it: on the averaging cases of the GPU
test, a model of the kernel's fp32 arithmetic (drq_ref.fp32_model) stays at least 5x below TAU against the float64
reference (|err| / scale per element), and each semantic slip the GPU test must catch -- only copy k = 0 averaged, the loss
not divided by M, the gradient weight without its 1 / M, m summed without the 1 / K -- moves some element at least 5x TAU."""
import numpy as np
import pytest
import torch

import c51_ref as C
import drq_ref as D

RB_ERR_INVAL, RB_ERR_RANGE = -22, -34
ONE = 8   # a pointer that is never dereferenced: validation fails first


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


def test_gather_aug_refusals_without_gpu():
    # frames, timestep, action, reward, nonterminal, size, data_idx, B, history, n, gamma_pow, states, next_states, actions,
    # returns, nonterminals, pad, intensity, m_copies, k_copies, seed, rng_counter, shifts, scales, stream
    good = [ONE] * 5 + [1000, ONE, 32, 4, 3] + [ONE] * 6 + [4, 0.05, 2, 2, 7, ONE, ONE, ONE, None]
    ptrs = [0, 1, 2, 3, 4, 6, 10, 11, 12, 13, 14, 15, 21, 22, 23]

    def call(**change):
        a = list(good)
        for i, v in change.items():
            a[int(i[1:])] = v
        return lib().rb_gather_aug(*a)

    for i in ptrs:
        assert call(**{f"a{i}": None}) == RB_ERR_INVAL, i
        assert b"null" in lib().rb_last_error()
    for pad in (-1, 17):
        assert call(a16=pad) == RB_ERR_RANGE, pad
    for s in (-0.01, 0.51, float("nan"), float("inf")):
        assert call(a17=s) == RB_ERR_RANGE, s
    for c in (0, 9):
        assert call(a18=c) == RB_ERR_RANGE and call(a19=c) == RB_ERR_RANGE, c
    assert call(a16=0, a17=0.0, a18=1, a19=1) == RB_ERR_INVAL, "the all-default gather is rb_gather"
    assert b"rb_gather" in lib().rb_last_error()
    assert call(a8=40, a9=30) == RB_ERR_RANGE            # window > RB_MAX_WINDOW (rb_gather's check)
    assert call(a7=65536) == RB_ERR_RANGE                # B > 65535
    for i in (5, 7, 8, 9):
        assert call(**{f"a{i}": 0}) == RB_ERR_INVAL, i   # sizes must be positive


def test_c51_avg_refusals_without_gpu():
    # z_online, z_target, A, Z, actions, returns, nonterminals, weights, support, vmin, vmax, delta_z, gamma_n, B, M, K,
    # loss, dz, m_out, astar_out, stream
    good = [ONE, ONE, 6, 51] + [ONE] * 5 + [-10.0, 10.0, 0.4, 0.97, 32, 2, 2, ONE, ONE, None, None, None]

    def call(**change):
        a = list(good)
        for i, v in change.items():
            a[int(i[1:])] = v
        return lib().rb_c51_dueling_avg_loss_grad(*a)

    for i in (0, 1, 4, 5, 6, 7, 8, 16, 17):
        assert call(**{f"a{i}": None}) == RB_ERR_INVAL, i
    for i, v in ((13, 0), (2, 0), (3, 1)):
        assert call(**{f"a{i}": v}) == RB_ERR_INVAL, (i, v)
    assert call(a3=129) == RB_ERR_RANGE
    for c in (0, 9):
        assert call(a14=c) == RB_ERR_RANGE and call(a15=c) == RB_ERR_RANGE, c
    assert call(a2=64, a3=128, a14=8, a15=8) == RB_ERR_RANGE   # (M + 2K) z rows do not fit in shared memory


def test_signatures_and_kernel_ids():
    from rainbow_b200 import _lib
    assert len(_lib.SIGNATURES["rb_gather_aug"][1]) == 25
    assert len(_lib.SIGNATURES["rb_c51_dueling_avg_loss_grad"][1]) == 21
    assert _lib.PROFILE_IDS[-2:] == ["gather_aug", "c51_dueling_avg"]
    assert _lib.PROFILE_IDS.index("gather_shift") == len(_lib.KERNEL_IDS) - 1


def test_replay_checks_before_cuda():
    from rainbow_b200.memory import ReplayMemory
    mem = ReplayMemory.__new__(ReplayMemory)
    mem.rng = "philox"
    assert mem._check_augmentation(0, 0.0, (1, 1)) == (0, 0.0, (1, 1))
    assert mem._check_augmentation(4, 0.05, (2, 8)) == (4, 0.05, (2, 8))
    for bad in ((17, 0.0, (1, 1)), (0, -0.01, (1, 1)), (0, 0.51, (1, 1)), (0, float("nan"), (1, 1)), (0, 0.0, (0, 1)),
                (0, 0.0, (1, 9))):
        with pytest.raises(ValueError):
            mem._check_augmentation(*bad)
    mem.rng = "numpy"
    assert mem._check_augmentation(0, 0.0, (1, 1)) == (0, 0.0, (1, 1))
    for bad in ((4, 0.0, (1, 1)), (0, 0.05, (1, 1)), (0, 0.0, (2, 1))):
        with pytest.raises(ValueError):
            mem._check_augmentation(*bad)


def test_multiplier_reference():
    """Box-Muller on philox_ref's words gives standard normals; the streams of different copies and sides differ; the
    clamped multipliers are fma(s, +-2, 1)."""
    from scipy import stats
    mult, n = D.multipliers(0x9E3779B97F4A7C15, (5 << 32) + 17, 20000, 2, 0.05)
    for side in (0, 1):
        for j in (0, 1):
            assert stats.kstest(n[side, j], "norm").pvalue > 1e-4
    assert abs(np.corrcoef(n[0, 0], n[1, 0])[0, 1]) < 0.05 and abs(np.corrcoef(n[0, 0], n[0, 1])[0, 1]) < 0.05
    assert mult.min() == pytest.approx(0.9) and mult.max() == pytest.approx(1.1)
    assert D.clamp_value(0.05, 1) == np.float32(1.1) and D.clamp_value(0.5, -1) == np.float32(0.0)
    assert D.aug_offsets(3, 9, 4, 0, 2).sum() == 0


# the averaging cases of tests/test_gpu_drq.py that the bound is sized on
AVG_CASES = [(32, 6, 51, "pm10", 2, 2), (5, 1, 2, "pm10", 1, 2), (33, 18, 51, "m3to7", 2, 1), (35, 6, 128, "0to20", 3, 2),
             (3, 18, 128, "pm10", 2, 2), (35, 6, 51, "pm10", 8, 8)]


def _rel(got, ref, sc):
    """max |got - ref| / scale; an element with scale 0 (weight 0) counts only if it differs."""
    return float(torch.nan_to_num((got - ref).abs() / sc, nan=0.0).max())


def _errors(inp, astar, m, loss, dz):
    m_ref, m_sc, _, ok = D.target(inp, astar)
    assert ok
    (l_ref, l_sc), _, (dz_ref, dz_sc) = D.loss_dz(inp, m)
    e = lambda got, ref, sc: _rel(got.double(), ref, sc)
    return e(m, m_ref, m_sc), e(loss, l_ref, l_sc), e(dz, dz_ref, dz_sc)


@pytest.mark.parametrize("case", AVG_CASES, ids=[f"B{c[0]}-A{c[1]}-Z{c[2]}-M{c[4]}-K{c[5]}" for c in AVG_CASES])
def test_tolerance_separates_fp32_arithmetic_from_semantic_slips(case):
    B, A, Z, sup, M, K = case
    inp = D.make_inputs(B, A, Z, sup, 11 + B + Z, M, K)
    astar, m, loss, dz = D.fp32_model(inp)
    model = max(_errors(inp, astar, m, loss, dz))
    assert np.isfinite(model) and model * 5 <= C.TAU, f"the fp32 model's largest error is {model:.3g} of the scale"

    m_ref, m_sc, ms, _ = D.target(inp, astar)
    (l_ref, l_sc), losses, (dz_ref, dz_sc) = D.loss_dz(inp, m_ref)
    rel = _rel
    slips = {}
    if B < 32:   # a handful of rows may all be terminal or clamped: every target copy then projects to the same m
        return
    if K > 1:
        slips["only k = 0 averaged"] = rel(ms[0], m_ref, m_sc)
        slips["m without 1 / K"] = rel(sum(ms), m_ref, m_sc)
    if M > 1:
        slips["loss not divided by M"] = rel(l_ref * M, l_ref, l_sc)
        slips["wi without 1 / M"] = rel(dz_ref * M, dz_ref, dz_sc)
    for name, v in slips.items():
        assert v >= 5 * C.TAU, f"{name}: {v:.3g}"
