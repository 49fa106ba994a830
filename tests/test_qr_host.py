"""Quantile regression (args.distribution = "quantile") without a GPU: the option checks, the host-side refusals of the four
C entry points with the library loaded, and tests/qr_ref.py's closed-form loss and gradient against torch autograd of the
objective."""
import argparse
import ctypes as C
import math

import pytest
import torch

import qr_ref as Q

RB_ERR_INVAL, RB_ERR_RANGE = -22, -34


def make_args(**kw):
    d = dict(device=torch.device("cpu"), history_length=4, discount=0.99, multi_step=3, priority_weight=0.4,
             priority_exponent=0.5, atoms=51, V_min=-10.0, V_max=10.0, batch_size=32, norm_clip=10.0, model=None,
             learning_rate=6.25e-5, adam_eps=1.5e-4, architecture="data-efficient", hidden_size=64, noisy_std=0.1)
    d.update(kw)
    return argparse.Namespace(**d)


# ---- options -------------------------------------------------------------------------------------------------------------
def test_distribution_options():
    from rainbow_b200.agent import distribution_options
    assert distribution_options(make_args()) == ("categorical", None)
    assert distribution_options(make_args(distribution=None, quantile_kappa=5.0)) == ("categorical", None)
    assert distribution_options(make_args(distribution="categorical")) == ("categorical", None)
    assert distribution_options(make_args(distribution="quantile")) == ("quantile", 1.0)
    assert distribution_options(make_args(distribution="quantile", quantile_kappa=None)) == ("quantile", 1.0)
    assert distribution_options(make_args(distribution="quantile", quantile_kappa=0.25)) == ("quantile", 0.25)
    assert distribution_options(make_args(distribution="quantile", atoms=2)) == ("quantile", 1.0)
    assert distribution_options(make_args(distribution="quantile", atoms=128)) == ("quantile", 1.0)


@pytest.mark.parametrize("bad", [dict(distribution="qr"), dict(distribution="Quantile"), dict(distribution=1),
                                 dict(distribution="quantile", quantile_kappa=0.0),
                                 dict(distribution="quantile", quantile_kappa=-1.0),
                                 dict(distribution="quantile", quantile_kappa=math.nan),
                                 dict(distribution="quantile", quantile_kappa=math.inf),
                                 dict(distribution="quantile", quantile_kappa=1e-50),    # 0 as an fp32
                                 dict(distribution="quantile", quantile_kappa=1e39),     # inf as an fp32
                                 dict(distribution="quantile", atoms=1), dict(distribution="quantile", atoms=129)])
def test_distribution_options_refuse(bad):
    from rainbow_b200.agent import distribution_options
    with pytest.raises(ValueError):
        distribution_options(make_args(**bad))


@pytest.mark.parametrize("copies", [dict(augment_m=2), dict(augment_k=2), dict(augment_m=2, augment_k=4)])
def test_quantile_refuses_drq_averaging(copies):
    """Agent.__init__ runs this check before it builds anything."""
    from rainbow_b200.agent import distribution_options
    with pytest.raises(ValueError, match="quantile"):
        distribution_options(make_args(distribution="quantile", **copies))
    assert distribution_options(make_args(**copies)) == ("categorical", None)
    assert distribution_options(make_args(distribution="quantile", augment_m=1, augment_k=1)) == ("quantile", 1.0)


def test_default_carries_no_quantile_state():
    from rainbow_b200.model import DQN
    net = DQN(make_args(), 4)
    assert net.quantile is False
    q = DQN(make_args(distribution="quantile"), 4)
    assert q.quantile is True
    # same parameters, same names: reset_table and redo_table apply as they are
    assert [(n, p.shape) for n, p in net.named_parameters()] == [(n, p.shape) for n, p in q.named_parameters()]
    assert list(net.state_dict()) == list(q.state_dict())


def test_quantile_forward_has_no_log_form():
    from rainbow_b200.model import DQN
    net = DQN(make_args(distribution="quantile", atoms=8), 3)
    net.use_fused_head = False
    x = torch.rand(2, 4, 84, 84)
    with torch.no_grad():
        q = net(x)
        assert q.shape == (2, 3, 8) and torch.equal(q, net.logits(x))
    with pytest.raises(ValueError):
        net(x, log=True)


# ---- C ABI refusals ------------------------------------------------------------------------------------------------------
def test_qr_abi_refusals_without_gpu():
    from rainbow_b200 import _lib
    L = _lib.load()
    one = C.c_void_p(8)  # never dereferenced: validation fails first

    def dueling(z=one, loss=one, dz=one, A=6, N=51, kappa=1.0, B=4):
        return L.rb_qr_dueling_loss_grad(z, one, A, N, one, one, one, one, kappa, 0.97, B, loss, dz, None, None, None)

    assert dueling(z=None) == RB_ERR_INVAL and b"null" in L.rb_last_error()
    assert dueling(loss=None) == RB_ERR_INVAL and dueling(dz=None) == RB_ERR_INVAL
    assert dueling(N=1) == RB_ERR_INVAL and dueling(N=129) == RB_ERR_RANGE and dueling(A=0) == RB_ERR_INVAL
    for k in (0.0, -1.0, math.nan, math.inf):
        assert dueling(kappa=k) == RB_ERR_INVAL and b"kappa" in L.rb_last_error()
    assert dueling(B=0) == RB_ERR_INVAL and dueling(B=-3) == RB_ERR_INVAL
    assert dueling(A=200, N=128) == RB_ERR_RANGE                 # (3 (N + A N) + 4 N + A) floats over 200 KB

    def plain(q=one, grad=one, A=6, N=51, kappa=1.0, B=4):
        return L.rb_qr_loss_grad(q, one, one, one, one, one, one, kappa, 0.97, B, A, N, one, grad, None, None, None)

    assert plain(q=None) == RB_ERR_INVAL and plain(grad=None) == RB_ERR_INVAL
    assert plain(N=1) == RB_ERR_INVAL and plain(N=129) == RB_ERR_RANGE
    for k in (0.0, -0.5, math.nan, -math.inf):
        assert plain(kappa=k) == RB_ERR_INVAL
    assert plain(B=0) == RB_ERR_INVAL and plain(A=0) == RB_ERR_INVAL

    assert L.rb_qr_q_values(None, 4, 6, 51, one, None, None, None) == RB_ERR_INVAL
    assert L.rb_qr_q_values(one, 4, 6, 51, None, None, None, None) == RB_ERR_INVAL      # no output requested
    assert L.rb_qr_q_values(one, 4, 6, 1, one, None, None, None) == RB_ERR_INVAL
    assert L.rb_qr_q_values(one, 4, 6, 129, one, None, None, None) == RB_ERR_RANGE
    assert L.rb_qr_q_values(one, 0, 6, 51, one, None, None, None) == RB_ERR_INVAL

    def stats(theta=one, z=one, q=None, B=4, N=51, scratch=one):
        return L.rb_learn_stats_batch_qr(one, one, one, theta, z, q, B, 6, N, scratch, None)

    assert stats(theta=None) == RB_ERR_INVAL and stats(scratch=None) == RB_ERR_INVAL
    assert stats(z=None) == RB_ERR_INVAL and stats(q=one) == RB_ERR_INVAL              # exactly one of z and q
    assert stats(N=1) == RB_ERR_INVAL and stats(N=129) == RB_ERR_RANGE and stats(B=0) == RB_ERR_INVAL


# ---- the reference against autograd -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,N,kappa", [(7, 2, 1.0), (9, 51, 0.25), (5, 128, 10.0), (12, 33, 1.0)])
def test_reference_is_autograd_of_the_objective(B, N, kappa):
    """qr_ref.quantile_loss_grad's closed form against torch autograd of (1/B) sum_b w_b loss_b, the loss written with
    torch's own Huber loss (huber_loss(delta=kappa) = H_kappa), on rows whose |u| straddles kappa, rows all inside and
    rows all outside, weights 0 and 1 included."""
    g = torch.Generator().manual_seed(B * N)
    theta = torch.randn(B, N, generator=g, dtype=torch.float64) * 2.0 * kappa
    T = torch.randn(B, N, generator=g, dtype=torch.float64) * 2.0 * kappa + 0.5 * kappa
    theta[1] = torch.rand(N, generator=g, dtype=torch.float64) * 0.2 * kappa             # every |u| < kappa
    T[1] = torch.rand(N, generator=g, dtype=torch.float64) * 0.2 * kappa
    T[2] = theta[2].max() + 2.0 * kappa + torch.rand(N, generator=g, dtype=torch.float64)  # every u > kappa
    w = torch.rand(B, generator=g, dtype=torch.float64)
    w[0], w[3] = 0.0, 1.0
    u = T.unsqueeze(1) - theta.unsqueeze(2)
    assert bool((u.abs() < kappa).any()) and bool((u.abs() > kappa).any())
    assert bool((u[1].abs() < kappa).all()) and bool((u[2] > kappa).all())

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
    assert bool((grad[0] == 0).all()), "weight 0: an exactly zero gradient"
    # the taus are the midpoints, and both sides of each quantile's weight sum to 1
    assert torch.equal(Q.taus(N), tau)
