"""DrQ's K / M averaging under the quantile loss without a GPU: the opt-in switch (args.quantile_average_copies), the
host-side refusals of rb_qr_dueling_avg_loss_grad and rb_qr_dueling_avg_vt_loss_grad (answered before any launch), their
signatures, and tests/qr_drq_ref.py -- Tbar then qr_ref.loss_grad per online copy, averaged -- against torch autograd
of the averaged objective."""
import ctypes
import math

import numpy as np
import pytest
import torch

import qr_drq_ref as QD
import qr_ref as Q
from test_qr_host import make_args

RB_ERR_INVAL, RB_ERR_RANGE = -22, -34
ONE = 8   # a pointer that is never dereferenced: validation fails first


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


# ---- the switch ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("copies", [dict(augment_m=2), dict(augment_k=2), dict(augment_m=2, augment_k=2),
                                    dict(augment_m=8, augment_k=8)])
def test_switch_admits_the_quantile_loss_with_copies(copies):
    from rainbow_b200.agent import distribution_options
    for off in (dict(), dict(quantile_average_copies=None), dict(quantile_average_copies=False)):
        with pytest.raises(ValueError, match="quantile_average_copies") as e:
            distribution_options(make_args(distribution="quantile", **copies, **off))
        assert "quantile" in str(e.value) and "augment_m" in str(e.value)
    for on in (True, np.bool_(True)):
        got = distribution_options(make_args(distribution="quantile", quantile_kappa=0.25, quantile_average_copies=on,
                                             **copies))
        assert got == ("quantile", 0.25), "the 2-tuple is unchanged"
    for bad in (1, "yes", 1.0):
        with pytest.raises(ValueError, match="bool"):
            distribution_options(make_args(distribution="quantile", quantile_average_copies=bad, **copies))


def test_switch_is_read_only_where_it_applies():
    """Categorical, or quantile with one copy of each: the switch (any value, even a malformed one) changes nothing."""
    from rainbow_b200.agent import distribution_options
    for v in (True, False, None, "not read"):
        assert distribution_options(make_args(quantile_average_copies=v)) == ("categorical", None)
        assert distribution_options(make_args(augment_m=2, augment_k=2, quantile_average_copies=v)) == ("categorical", None)
        assert distribution_options(make_args(distribution="quantile", quantile_average_copies=v)) == ("quantile", 1.0)
        assert distribution_options(make_args(distribution="quantile", augment_m=1, augment_k=1,
                                              quantile_average_copies=v)) == ("quantile", 1.0)


# ---- the C entry points ------------------------------------------------------------------------------------------------------
def test_signatures():
    from rainbow_b200 import _lib
    assert len(_lib.SIGNATURES["rb_qr_dueling_avg_loss_grad"][1]) == 18
    assert len(_lib.SIGNATURES["rb_qr_dueling_avg_vt_loss_grad"][1]) == 19
    # rb_qr_dueling(_vt)_loss_grad's arguments with M, K after B
    for name in ("rb_qr_dueling_loss_grad", "rb_qr_dueling_vt_loss_grad"):
        base = _lib.SIGNATURES[name][1]
        avg = _lib.SIGNATURES[name.replace("dueling", "dueling_avg")][1]
        assert avg == base[:11] + [ctypes.c_int32, ctypes.c_int32] + base[11:]
    assert _lib.PROFILE_IDS[-2:] == ["gather_aug", "c51_dueling_avg"], "no new profile slot: RB_K_C51_DUELING_AVG"


@pytest.mark.parametrize("vt", [False, True], ids=["plain", "vt"])
def test_refusals_without_gpu(vt):
    # z_online, z_target, A, N, actions, returns, nonterminals, weights, kappa, gamma_n, B, M, K, loss, dz, theta_out,
    # astar_out, [eps,] stream
    good = [ONE, ONE, 6, 51] + [ONE] * 4 + [1.0, 0.97, 32, 2, 2, ONE, ONE, None, None] + ([1e-3] if vt else []) + [None]
    fn = lib().rb_qr_dueling_avg_vt_loss_grad if vt else lib().rb_qr_dueling_avg_loss_grad

    def call(**change):
        a = list(good)
        for i, v in change.items():
            a[int(i[1:])] = v
        return fn(*a)

    for i in (0, 1, 4, 5, 6, 7, 13, 14):
        assert call(**{f"a{i}": None}) == RB_ERR_INVAL, i
        assert b"null" in lib().rb_last_error()
    for i, v in ((10, 0), (10, -3), (2, 0), (3, 1)):
        assert call(**{f"a{i}": v}) == RB_ERR_INVAL, (i, v)
    for k in (0.0, -1.0, math.nan, math.inf):
        assert call(a8=k) == RB_ERR_INVAL and b"kappa" in lib().rb_last_error(), k
    assert call(a3=129) == RB_ERR_RANGE
    for c in (0, 9, -1):
        assert call(a11=c) == RB_ERR_RANGE and call(a12=c) == RB_ERR_RANGE, c
        assert b"copies" in lib().rb_last_error()
    assert call(a2=64, a3=128, a11=8, a12=8) == RB_ERR_RANGE   # (M + 2K) z rows do not fit in shared memory
    assert b"too large" in lib().rb_last_error()
    if vt:
        for e in (-1e-3, 1.5, math.nan):
            assert call(a17=e) == RB_ERR_INVAL and b"eps" in lib().rb_last_error(), e


# ---- the reference against autograd ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,A,N,kappa,M,K,eps", [(12, 6, 51, 1.0, 2, 2, None), (7, 1, 2, 0.25, 3, 5, None),
                                                 (13, 18, 33, 10.0, 2, 1, None), (6, 3, 128, 1.0, 1, 2, None),
                                                 (12, 6, 65, 1.0, 2, 2, 1e-3), (7, 2, 8, 0.25, 8, 8, 0.0)])
def test_reference_is_autograd_of_the_averaged_objective(B, A, N, kappa, M, K, eps):
    """qr_drq_ref's Tbar-then-closed-form loss and dz rows against torch autograd of the averaged objective, written from
    the definition (theta of every online copy through the dueling combination, u against the mean of the K target rows);
    rows of weight 0 have an exactly zero gradient; at M = K = 1 the reference is qr_ref's."""
    inp = QD.make_inputs(B, A, N, kappa, 100 * B + N, M, K, eps)
    astar = torch.stack([QD.means(QD.single(inp, 0, k))[0].argmax(1) for k in range(K)])
    Tbar, _, Ts, ok = QD.target(inp, astar)
    assert ok
    (loss, _), losses, (dz, _) = QD.loss_dz(inp, Tbar)

    z = inp["z_on"].double().requires_grad_()
    loss_ag, obj = QD.objective(dict(inp, z_on=z), astar)
    obj.backward()
    assert torch.allclose(loss, loss_ag.detach(), rtol=1e-12, atol=1e-14)
    assert torch.allclose(dz, z.grad[:M * B], rtol=1e-10, atol=1e-15)
    assert bool((z.grad[M * B:] == 0).all()), "no gradient through the target copies"
    zero_w = inp["weights"] == 0
    assert bool(zero_w.any()) and bool((dz.view(M, B, -1)[:, zero_w] == 0).all())
    if K > 1:
        assert not torch.equal(Ts[0], Ts[1]), "the copies differ, so the average is not a copy"

    one = dict(inp, M=1, K=1, z_on=torch.cat([inp["z_on"][:B], inp["z_on"][M * B:(M + 1) * B]]), z_tg=inp["z_tg"][:B])
    T1, s1, _, _ = QD.target(one, astar[:1])
    T0, s0 = (Q.targets if eps is None else QD.V.qr_targets)(QD.single(inp), astar[0])
    assert torch.equal(T1, T0) and torch.allclose(s1, s0, rtol=QD.U / Q.TAU * 2, atol=0)


def test_slips_move_elements_past_the_tolerance():
    """Each slip of the definition the GPU test must catch moves some element by at least 5 x TAU of its scale."""
    B, A, N, kappa, M, K = 42, 6, 51, 1.0, 2, 2
    inp = QD.make_inputs(B, A, N, kappa, 3, M, K)
    astar = torch.stack([QD.means(QD.single(inp, 0, k))[0].argmax(1) for k in range(K)])
    Tbar, tsc, Ts, _ = QD.target(inp, astar)
    (loss, lsc), _, (dz, dsc) = QD.loss_dz(inp, Tbar)
    rel = lambda got, ref, sc: float(torch.nan_to_num((got - ref).abs() / sc, nan=0.0).max())
    slips = {
        "a*_0 for every copy": rel(QD.target(inp, torch.stack([astar[0]] * K))[0], Tbar, tsc),
        "only copy 0": rel(Ts[0], Tbar, tsc),
        "Tbar without 1 / K": rel(sum(Ts), Tbar, tsc),
        "loss not divided by M": rel(loss * M, loss, lsc),
        "wi = w / B": rel(dz * M, dz, dsc),
    }
    for name, v in slips.items():
        assert v >= 5 * Q.TAU, f"{name}: {v:.3g}"
    # under value rescaling: the average taken of h^-1(T_k) and mapped back by h, instead of in h units
    vin = QD.make_inputs(B, A, N, kappa, 3, M, K, eps=1e-3)
    va = torch.stack([QD.means(QD.single(vin, 0, k))[0].argmax(1) for k in range(K)])
    vT, vsc, vTs, _ = QD.target(vin, va)
    after = QD.V.h(sum(QD.V.hinv(t, 1e-3) for t in vTs) / K, 1e-3)
    assert rel(after, vT, vsc) >= 5 * Q.TAU


def test_mean_of_tbar_is_the_mean_of_the_averaged_target_values():
    """The definition's point 3: mean_n Tbar_n = (1 / K) sum_k mean_n T_k,n, the Q target of DrQ's Algorithm 1."""
    inp = QD.make_inputs(33, 6, 51, 1.0, 9, 1, 4)
    astar = torch.stack([QD.means(QD.single(inp, 0, k))[0].argmax(1) for k in range(4)])
    Tbar, _, Ts, _ = QD.target(inp, astar)
    assert torch.allclose(Tbar.mean(1), sum(t.mean(1) for t in Ts) / 4, rtol=1e-14, atol=1e-14)
