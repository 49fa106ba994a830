"""Value rescaling (args.value_transform = "rescale") without a GPU: the option checks, the default path's lack of transform
state, the float64 forms of h and h^-1 of tests/vt_ref.py against independent evaluations, the host-side refusals of the
seven C entry points with the library loaded, and the reference's transformed quantile objective against torch
autograd."""
import argparse
import ctypes as C
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

import qr_ref as Q
import vt_ref as V

RB_ERR_INVAL, RB_ERR_RANGE = -22, -34


def make_args(**kw):
    d = dict(device=torch.device("cpu"), history_length=4, discount=0.99, multi_step=3, priority_weight=0.4,
             priority_exponent=0.5, atoms=51, V_min=-10.0, V_max=10.0, batch_size=32, norm_clip=10.0, model=None,
             learning_rate=6.25e-5, adam_eps=1.5e-4, architecture="data-efficient", hidden_size=64, noisy_std=0.1)
    d.update(kw)
    return argparse.Namespace(**d)


# ---- options -------------------------------------------------------------------------------------------------------------
def test_value_transform_options():
    from rainbow_b200.agent import value_transform_options as opt
    assert opt(make_args()) == (None, None)
    assert opt(make_args(value_transform=None, value_transform_eps=0.5)) == (None, None)
    assert opt(make_args(value_transform="none")) == (None, None)
    e3 = float(np.float32(1e-3))          # eps is kept as the fp32 the kernels take
    assert opt(make_args(value_transform="rescale")) == ("rescale", e3)
    assert opt(make_args(value_transform="rescale", value_transform_eps=None)) == ("rescale", e3)
    assert opt(make_args(value_transform="rescale", value_transform_eps=1e-2)) == ("rescale", float(np.float32(1e-2)))
    assert opt(make_args(value_transform="rescale", value_transform_eps=0.0)) == ("rescale", 0.0)
    assert opt(make_args(value_transform="rescale", value_transform_eps=0.25)) == ("rescale", 0.25)
    assert opt(make_args(value_transform="rescale", value_transform_eps=1)) == ("rescale", 1.0)
    assert opt(make_args(value_transform="rescale", value_transform_eps=np.float32(1e-3))) == ("rescale", e3)
    tiny = float(np.finfo(np.float32).tiny)
    assert opt(make_args(value_transform="rescale", value_transform_eps=tiny)) == ("rescale", tiny)


@pytest.mark.parametrize("bad", [dict(value_transform="Rescale"), dict(value_transform="h"), dict(value_transform=1),
                                 dict(value_transform=True),
                                 dict(value_transform="rescale", value_transform_eps=-1e-3),
                                 dict(value_transform="rescale", value_transform_eps=1.5),
                                 dict(value_transform="rescale", value_transform_eps=math.nan),
                                 dict(value_transform="rescale", value_transform_eps=math.inf),
                                 dict(value_transform="rescale", value_transform_eps=1.0 + 1e-12),
                                 dict(value_transform="rescale", value_transform_eps=1e-50),   # 0 as an fp32
                                 dict(value_transform="rescale", value_transform_eps=1e-40),   # subnormal fp32
                                 dict(value_transform="rescale", value_transform_eps="0.001"),
                                 dict(value_transform="rescale", value_transform_eps=True)])
def test_value_transform_options_refuse(bad):
    from rainbow_b200.agent import value_transform_options
    with pytest.raises(ValueError):
        value_transform_options(make_args(**bad))


def test_agent_checks_before_building():
    """Agent.__init__ refuses a bad option before it needs a device (here: a CPU device it would refuse later)."""
    from rainbow_b200 import _lib
    from rainbow_b200.agent import Agent

    class Env:
        def action_space(self):
            return 4

    with pytest.raises(_lib.RainbowB200Error):
        Agent(make_args(value_transform="rescale"), Env())      # the option is fine: the device check refuses
    args = make_args(value_transform="bad", device=torch.device("cuda:0"))
    with pytest.raises(ValueError, match="value_transform"):
        Agent(args, Env())


def test_default_carries_no_transform_state():
    """The default path: the checkpoint writer records nothing, the loss wrappers get eps None (the plain entries)."""
    import rainbow_b200.agent as agent_mod
    a = object.__new__(agent_mod.Agent)
    a.value_transform, a.value_transform_eps = agent_mod.value_transform_options(make_args())
    a.support = a.q_support = torch.zeros(3)
    assert a._vt_args() == dict(support_q=None, eps=None)
    assert a.value_transform is None and a.value_transform_eps is None


# ---- h and h^-1 in float64 -------------------------------------------------------------------------------------------------
def _grid():
    y = torch.cat([torch.logspace(-30, 6, 721, dtype=torch.float64), torch.tensor([0.0, 1.0, 3.0], dtype=torch.float64)])
    return torch.cat([y, -y])


@pytest.mark.parametrize("eps", [0.0, 1e-3, 1e-2, 1.0])
def test_round_trip_and_oddness(eps):
    y = _grid()
    assert torch.allclose(V.h(V.hinv(y, eps), eps), y, rtol=4e-15, atol=0.0)
    assert torch.allclose(V.hinv(V.h(y, eps), eps), y, rtol=4e-15, atol=0.0)
    assert torch.equal(V.h(-y, eps), -V.h(y, eps)) and torch.equal(V.hinv(-y, eps), -V.hinv(y, eps))
    assert bool((V.h(y[1:], eps) > V.h(y[:-1], eps)).sum() > 0)
    pos = y[y > 0].sort().values
    assert bool((V.h(pos[1:], eps) >= V.h(pos[:-1], eps)).all()), "h is monotone"


def test_eps_zero_closed_form():
    y = _grid()
    assert torch.allclose(V.hinv(y, 0.0), y.sign() * y.abs() * (y.abs() + 2.0), rtol=1e-15, atol=0.0)
    x = _grid()
    x = x[x.abs() >= 1e-3]      # where the textbook sqrt(|x| + 1) - 1 does not cancel in float64
    assert torch.allclose(V.h(x, 0.0), x.sign() * ((x.abs() + 1.0).sqrt() - 1.0), rtol=1e-12, atol=0.0)


@pytest.mark.parametrize("eps", [1e-3, 1e-2, 1.0])
def test_inverse_against_textbook_where_it_is_accurate(eps):
    """For |y| >= 1 the textbook inverse loses at most a few digits in float64: agreement to 1e-12 relative."""
    y = torch.logspace(0, 6, 301, dtype=torch.float64)
    y = torch.cat([y, -y])
    assert torch.allclose(V.hinv(y, eps), V.hinv_textbook(y, eps), rtol=1e-12, atol=0.0)


def _h_exact_bracket(x, eps):
    """h(x) for x >= 0 rational, bracketed: sqrt(x + 1) by Fractions on both sides (bisection to 2^-80 relative)."""
    s = Fraction(x) + 1
    lo, hi = Fraction(1), s
    for _ in range(200):
        mid = (lo + hi) / 2
        if mid * mid <= s:
            lo = mid
        else:
            hi = mid
        if hi - lo <= lo / 2 ** 80:
            break
    e = Fraction(eps)
    return Fraction(x) / (hi + 1) + e * Fraction(x), Fraction(x) / (lo + 1) + e * Fraction(x)


@pytest.mark.parametrize("eps", [0.0, 1e-3, 1e-2, 1.0])
def test_inverse_for_small_y_by_the_defining_equation(eps):
    """Small |y|: h(x) = x / 2 + eps x + O(x^2), so h^-1(y) = 2y / (1 + 2 eps) + O(y^2); and x = h^-1(y) solves y = h(x):
    h at x (1 -+ 1e-13), evaluated in exact rational arithmetic, brackets y."""
    for y in (1e-30, 1e-20, 1e-12, 1e-8, 1e-6, 1e-4):
        x = float(V.hinv(torch.tensor(y, dtype=torch.float64), eps))
        assert abs(x - 2 * y / (1 + 2 * eps)) <= 2 * y * y + 1e-15 * y
        h_lo = _h_exact_bracket(x * (1 - 1e-13), eps)[1]
        h_hi = _h_exact_bracket(x * (1 + 1e-13), eps)[0]
        assert h_lo < Fraction(y) < h_hi, (y, eps)


def test_textbook_inverse_cancels():
    """Why the kernel may not use it: fp32-sized relative error already at |y| ~ 1e-6 in float64 with eps = 1e-3."""
    y = torch.tensor([1e-6, 1e-9], dtype=torch.float64)
    rel = ((V.hinv_textbook(y, 1e-3) - V.hinv(y, 1e-3)) / V.hinv(y, 1e-3)).abs()
    assert bool((rel > 1e-8).all())


# ---- C ABI refusals ------------------------------------------------------------------------------------------------------
def test_vt_abi_refusals_without_gpu():
    from rainbow_b200 import _lib
    L = _lib.load()
    one = C.c_void_p(8)  # never dereferenced: validation fails first
    bad_eps = (-1e-3, 1.5, math.nan, math.inf, -math.inf)

    def c51(sq=one, sup=one, eps=1e-3, Z=51):
        return L.rb_c51_vt_loss_grad(one, one, one, one, one, one, one, sup, -10.0, 10.0, 0.4, 0.97, 4, 6, Z, one, one,
                                     None, None, sq, eps, None)

    def duel(sq=one, sup=one, eps=1e-3, Z=51):
        return L.rb_c51_dueling_vt_loss_grad(one, one, 6, Z, one, one, one, one, sup, -10.0, 10.0, 0.4, 0.97, 4, one, one,
                                             None, None, sq, eps, None)

    def avg(sq=one, sup=one, eps=1e-3, Z=51, M=2):
        return L.rb_c51_dueling_avg_vt_loss_grad(one, one, 6, Z, one, one, one, one, sup, -10.0, 10.0, 0.4, 0.97, 4, M, 2,
                                                 one, one, None, None, sq, eps, None)

    for f in (c51, duel, avg):
        assert f(sq=None) == RB_ERR_INVAL and b"null" in L.rb_last_error()
        assert f(sup=None) == RB_ERR_INVAL
        for e in bad_eps:
            assert f(eps=e) == RB_ERR_INVAL and b"eps" in L.rb_last_error()
        assert f(Z=1) == RB_ERR_INVAL and f(Z=129) == RB_ERR_RANGE
    assert avg(M=0) == RB_ERR_RANGE

    def qrd(z=one, eps=1e-3, N=51, kappa=1.0):
        return L.rb_qr_dueling_vt_loss_grad(z, one, 6, N, one, one, one, one, kappa, 0.97, 4, one, one, None, None, eps,
                                            None)

    def qrp(q=one, eps=1e-3, N=51, kappa=1.0):
        return L.rb_qr_vt_loss_grad(q, one, one, one, one, one, one, kappa, 0.97, 4, 6, N, one, one, None, None, eps, None)

    for f, k in ((qrd, "z"), (qrp, "q")):
        assert f(**{k: None}) == RB_ERR_INVAL
        for e in bad_eps:
            assert f(eps=e) == RB_ERR_INVAL
        assert f(N=1) == RB_ERR_INVAL and f(N=129) == RB_ERR_RANGE and f(kappa=0.0) == RB_ERR_INVAL

    assert L.rb_qr_vt_q_values(None, 4, 6, 51, one, None, None, 1e-3, None) == RB_ERR_INVAL
    assert L.rb_qr_vt_q_values(one, 4, 6, 51, None, None, None, 1e-3, None) == RB_ERR_INVAL
    assert L.rb_qr_vt_q_values(one, 4, 6, 129, one, None, None, 1e-3, None) == RB_ERR_RANGE
    for e in bad_eps:
        assert L.rb_qr_vt_q_values(one, 4, 6, 51, one, None, None, e, None) == RB_ERR_INVAL

    def stats(theta=one, z=one, q=None, N=51, eps=1e-3):
        return L.rb_learn_stats_batch_qr_vt(one, one, one, theta, z, q, 4, 6, N, one, eps, None)

    assert stats(theta=None) == RB_ERR_INVAL and stats(z=None) == RB_ERR_INVAL and stats(q=one) == RB_ERR_INVAL
    assert stats(N=129) == RB_ERR_RANGE
    for e in bad_eps:
        assert stats(eps=e) == RB_ERR_INVAL


# ---- the reference's transformed objective against autograd ---------------------------------------------------------------
@pytest.mark.parametrize("B,N,kappa,eps", [(7, 2, 1.0, 1e-3), (9, 51, 0.25, 0.0), (5, 128, 10.0, 1e-2)])
def test_transformed_objective_is_autograd(B, N, kappa, eps):
    """The loss through vt_ref's targets T = h(r + s h^-1(theta')) against torch autograd of the same objective built
    from the textbook-free float64 h / h^-1: the gradient flows through theta only (T is a constant target)."""
    g = torch.Generator().manual_seed(B * N)
    theta = torch.randn(B, N, generator=g, dtype=torch.float64) * 3.0
    theta_t = torch.randn(B, N, generator=g, dtype=torch.float64) * 3.0
    r = (torch.rand(B, generator=g, dtype=torch.float64) * 2 - 1) * 1e3
    s = torch.full((B,), 0.97, dtype=torch.float64)
    s[0] = 0.0
    w = torch.rand(B, generator=g, dtype=torch.float64)
    T = V.h(r.unsqueeze(1) + s.unsqueeze(1) * V.hinv(theta_t, eps), eps)
    assert torch.allclose(T[0], V.h(r[0].expand(N), eps), rtol=0, atol=0)
    th = theta.clone().requires_grad_()
    uu = T.unsqueeze(1) - th.unsqueeze(2)
    tau = (torch.arange(N, dtype=torch.float64) + 0.5) / N
    weight = (tau.view(1, N, 1) - (uu.detach() < 0).double()).abs()
    huber = torch.nn.functional.huber_loss(T.unsqueeze(1).expand_as(uu), th.unsqueeze(2).expand_as(uu), reduction="none",
                                           delta=kappa)
    loss_ag = (weight * huber).sum(1).mean(1) / kappa
    ((w * loss_ag).sum() / B).backward()
    loss, grad = Q.quantile_loss_grad(theta, T, w, B, kappa)
    assert torch.allclose(loss, loss_ag.detach(), rtol=1e-12, atol=1e-14)
    assert torch.allclose(grad, th.grad, rtol=1e-12, atol=1e-15)
