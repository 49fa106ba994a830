"""The annealed horizon without a GPU: every refusal of rb_horizon_advance and rb_gather_horizon (answered before any
launch), the option checks, the checkpoint's horizon_step check, and the host table against tests/horizon_ref.py."""
import argparse
import math

import numpy as np
import pytest

import horizon_ref as HR

RB_ERR_INVAL, RB_ERR_RANGE = -22, -34
ONE = 4096   # a pointer that is never dereferenced: validation fails first


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


def args(**kw):
    d = dict(multi_step=3, discount=0.99, history_length=4)
    d.update(kw)
    return argparse.Namespace(**d)


# ---- entry points ------------------------------------------------------------------------------------------------------
def test_horizon_advance_refusals_without_gpu():
    L = lib()
    assert L.rb_horizon_advance(None, 4, ONE, ONE, None) == RB_ERR_INVAL
    assert L.rb_horizon_advance(ONE, 4, None, ONE, None) == RB_ERR_INVAL
    assert L.rb_horizon_advance(ONE, 4, ONE, None, None) == RB_ERR_INVAL
    for T in (0, -1, 65537, 2 ** 31 - 1):
        assert L.rb_horizon_advance(ONE, T, ONE, ONE, None) == RB_ERR_RANGE, T
        assert b"T outside" in L.rb_last_error()


def gather_call(n_max=10, history=4, B=8, size=1024, current=ONE, pad=0, intensity=0.0, M=1, K=1, counter=ONE, shifts=ONE,
                scales=ONE, frames=ONE):
    return lib().rb_gather_horizon(frames, ONE, ONE, ONE, ONE, size, ONE, B, history, n_max, current, ONE, ONE, ONE, ONE, ONE,
                                   pad, intensity, M, K, 1, counter, shifts, scales, None)


def test_gather_horizon_refusals_without_gpu():
    assert gather_call(current=None) == RB_ERR_INVAL
    assert gather_call(frames=None) == RB_ERR_INVAL
    assert gather_call(n_max=0) == RB_ERR_INVAL and gather_call(B=0) == RB_ERR_INVAL
    assert gather_call(n_max=61) == RB_ERR_RANGE and gather_call(history=60, n_max=5) == RB_ERR_RANGE
    assert gather_call(B=65536) == RB_ERR_RANGE
    for pad in (-1, 17):
        assert gather_call(pad=pad) == RB_ERR_RANGE
    for s in (-0.1, 0.51, float("nan"), float("inf")):
        assert gather_call(intensity=s) == RB_ERR_RANGE
    for M, K in ((0, 1), (1, 0), (9, 1), (1, 9)):
        assert gather_call(M=M, K=K) == RB_ERR_RANGE
    assert gather_call(pad=4, counter=None) == RB_ERR_INVAL and gather_call(pad=4, shifts=None) == RB_ERR_INVAL
    assert gather_call(intensity=0.05, scales=None) == RB_ERR_INVAL and gather_call(M=2, scales=None) == RB_ERR_INVAL


def test_signatures():
    from rainbow_b200 import _lib
    assert len(_lib.SIGNATURES["rb_horizon_advance"][1]) == 5 and len(_lib.SIGNATURES["rb_gather_horizon"][1]) == 25


def test_row_layout_is_rb_horizon():
    import ctypes as C

    from rainbow_b200 import _lib
    from rainbow_b200.horizon import ROW_DTYPE
    assert C.sizeof(_lib.Horizon) == ROW_DTYPE.itemsize == 264
    assert _lib.Horizon.gamma_n.offset == ROW_DTYPE.fields["gamma_n"][1] == 4
    assert _lib.Horizon.gamma_pow.offset == ROW_DTYPE.fields["gamma_pow"][1] == 8


# ---- options -----------------------------------------------------------------------------------------------------------
def test_options_off_by_default():
    from rainbow_b200.horizon import horizon_options
    assert horizon_options(args()) is None
    assert horizon_options(args(anneal_steps=0)) is None and horizon_options(args(anneal_steps=None)) is None
    assert horizon_options(args(anneal_steps=0, multi_step_start=3, discount_start=0.99)) is None
    assert horizon_options(args(anneal_steps=4)) == (4, 3, 3, 0.99, 0.99)
    assert horizon_options(args(anneal_steps=10000, multi_step_start=10, discount_start=0.97, discount=0.997)) == \
        (10000, 10, 3, 0.97, 0.997)


@pytest.mark.parametrize("bad", [dict(anneal_steps=65537), dict(anneal_steps=-1), dict(anneal_steps=2.5),
                                 dict(anneal_steps=True), dict(anneal_steps=3, multi_step_start=0),
                                 dict(anneal_steps=3, multi_step_start=2.5), dict(anneal_steps=3, discount_start=1.0),
                                 dict(anneal_steps=3, discount_start=0.9, discount=1.0),
                                 dict(anneal_steps=3, discount_start=float("nan")), dict(anneal_steps=3, discount_start=-0.1),
                                 dict(multi_step_start=5), dict(discount_start=0.9)])
def test_option_refusals(bad):
    from rainbow_b200.horizon import horizon_options
    with pytest.raises(ValueError):
        horizon_options(args(**bad))


def test_constant_discount_of_one_is_allowed():
    from rainbow_b200.horizon import horizon_options
    assert horizon_options(args(anneal_steps=3, multi_step_start=5, discount=1.0)) == (3, 5, 3, 1.0, 1.0)


# ---- the table ---------------------------------------------------------------------------------------------------------
SCHEDULES = [(10000, 10, 3, 0.97, 0.997), (6, 10, 3, 0.97, 0.997), (1, 10, 3, 0.97, 0.997), (7, 3, 3, 0.99, 0.99),
             (5, 1, 20, 0.9, 0.999), (17, 4, 4, 0.97, 0.997), (12, 60, 1, 0.5, 0.5), (65536, 2, 3, 0.99, 0.995)]


@pytest.mark.parametrize("sched", SCHEDULES, ids=[f"T{s[0]}-n{s[1]}-{s[2]}-g{s[3]}-{s[4]}" for s in SCHEDULES])
def test_table_is_the_reference(sched):
    from rainbow_b200.horizon import horizon_at, horizon_table
    T, n0, n1, g0, g1 = sched
    rows = horizon_table(*sched)
    assert rows.shape == (T + 1,)
    us = range(T + 1) if T <= 20000 else list(range(0, T + 1, 97)) + [1, T - 1, T]
    for u in us:
        n, gn, pw = HR.row(u, *sched)
        assert horizon_at(u, *sched) == HR.schedule(u, *sched)
        assert rows["n"][u] == n and rows["gamma_n"][u].tobytes() == gn.tobytes(), u
        assert rows["gamma_pow"][u].tobytes() == pw.tobytes(), u
        assert (rows["gamma_pow"][u, n:] == 0).all()
    assert (rows["n"][0], rows["n"][-1]) == (n0, n1)
    assert horizon_at(0, *sched) == (n0, g0) and horizon_at(T, *sched) == (n1, g1) and horizon_at(T + 5, *sched) == (n1, g1)
    d = np.diff(rows["n"].astype(np.int64))
    assert (d <= 0).all() if n1 <= n0 else (d >= 0).all(), "n moves monotonically"
    if g0 == g1:
        assert all(horizon_at(u, *sched)[1] == g0 for u in us)
    if n0 == n1:
        assert (rows["n"] == n0).all()


def test_half_even_at_ties():
    """Python's round() and the reference's exact rational rounding agree on ties and near them."""
    from rainbow_b200 import horizon as H
    for x in (0.5, 1.5, 2.5, 3.5, 4.5, 9.5, 2.4999999999999996, 2.5000000000000004):
        assert round(x) == HR.round_half_even(x)
    # a schedule whose midpoint lands on a tie: n from 2 to 8 passes exp(log 2 + f log 4) = 4 at f = 1/2, and 3 / 5 ...
    hits = [H.horizon_at(u, 8, 2, 8, 0.9, 0.9)[0] for u in range(9)]
    assert hits == [HR.schedule(u, 8, 2, 8, 0.9, 0.9)[0] for u in range(9)]
    assert hits[4] == 4


def test_bbf_ends_and_midpoint():
    from rainbow_b200.horizon import horizon_at
    assert horizon_at(0, 10000, 10, 3, 0.97, 0.997) == (10, 0.97)
    assert horizon_at(10000, 10000, 10, 3, 0.97, 0.997) == (3, 0.997)
    n, g = horizon_at(5000, 10000, 10, 3, 0.97, 0.997)
    assert n == round(math.sqrt(30)) and math.isclose(1 - g, math.sqrt(0.03 * 0.003), rel_tol=1e-12)


def test_replay_window_is_n_max(monkeypatch):
    """ReplayMemory reads multi_step_start: its n (the sampler's window) is max(n0, n1) with annealing on."""
    import torch

    from rainbow_b200 import memory as M
    monkeypatch.setattr(M, "_require_cuda", lambda d: torch.device("cpu"))
    monkeypatch.setattr(M, "SegmentTree", lambda *a: None)
    monkeypatch.setattr(M._lib, "load", lambda: None)
    kw = dict(device="cpu", history_length=4, priority_weight=0.4, priority_exponent=0.5, discount=0.997)
    for (a, want) in ((dict(multi_step=3), 3), (dict(multi_step=3, anneal_steps=6, multi_step_start=10), 10),
                      (dict(multi_step=3, anneal_steps=6), 3), (dict(multi_step=10, anneal_steps=6, multi_step_start=3), 10),
                      (dict(multi_step=3, multi_step_start=3), 3)):
        mem = M.ReplayMemory(argparse.Namespace(**kw, **a), 64, seed=1)
        assert mem.n == want, a
        assert mem.n_step_scaling.numel() == want
    with pytest.raises(ValueError):
        M.ReplayMemory(argparse.Namespace(**kw, multi_step=3, anneal_steps=6, multi_step_start=61), 64, seed=1)


# ---- checkpoint scalars --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("v,ok", [(None, True), (0, True), (5, True), (2 ** 63 - 1, True), (-1, False), (2 ** 63, False),
                                  (1.0, False), (True, False), ("3", False)])
def test_checkpoint_horizon_step_check(v, ok):
    from rainbow_b200 import checkpoint
    check = checkpoint._SCALARS[("learner", "horizon_step")]
    assert bool(check(v, None)) == ok
