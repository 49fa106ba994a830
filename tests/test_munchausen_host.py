"""Munchausen targets under the quantile loss without a GPU: the options (args.munchausen and its three parameters) and
every refusal, the C entries' signatures against the header and their host-side refusals, and tests/munchausen_ref.py --
its gradient against autograd, its limits (one action, alpha 0, tau -> 0) and the derivation of T's error scale against
an fp32 emulation of the kernel's arithmetic."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

import c51_ref as C
import munchausen_ref as MR
import qr_ref as Q
from test_qr_host import make_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RB_ERR_INVAL, RB_ERR_RANGE = -22, -34
ONE = 8   # a pointer that is never dereferenced: validation fails first
QR = dict(distribution="quantile")


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


# ---- options ---------------------------------------------------------------------------------------------------------------
def test_defaults_and_off():
    from rainbow_b200.agent import munchausen_options
    for off in (dict(), dict(munchausen=None), dict(munchausen=False), dict(munchausen=np.bool_(False))):
        assert munchausen_options(make_args(**QR, **off)) is None
        assert munchausen_options(make_args(**off)) is None, "off: nothing else is read"
    assert munchausen_options(make_args(munchausen=False, munchausen_alpha="not read")) is None
    got = munchausen_options(make_args(munchausen=True, **QR))
    assert got == (float(np.float32(0.9)), float(np.float32(0.03)), -1.0)
    got = munchausen_options(make_args(munchausen=np.bool_(True), munchausen_alpha=0, munchausen_temperature=1,
                                       munchausen_clip=-0.5, **QR))
    assert got == (0.0, 1.0, -0.5), "alpha = 0 (the soft target without the bonus) is allowed"
    assert munchausen_options(make_args(munchausen=True, munchausen_alpha=None, **QR))[0] == float(np.float32(0.9))


@pytest.mark.parametrize("bad", [1, "yes", 1.0])
def test_switch_must_be_a_bool(bad):
    from rainbow_b200.agent import munchausen_options
    with pytest.raises(ValueError, match="munchausen must be a bool"):
        munchausen_options(make_args(munchausen=bad, **QR))


@pytest.mark.parametrize("key,bad", [("munchausen_alpha", v) for v in (-0.1, 1.5, math.nan, math.inf, "0.5", True)] +
                         [("munchausen_temperature", v) for v in (0.0, -0.03, math.nan, math.inf, 1e-40, 1e39)] +
                         [("munchausen_clip", v) for v in (0.0, 1.0, math.nan, -math.inf, -1e39)])
def test_bad_parameters_are_refused(key, bad):
    from rainbow_b200.agent import munchausen_options
    with pytest.raises(ValueError, match=key):
        munchausen_options(make_args(munchausen=True, **{key: bad}, **QR))


@pytest.mark.parametrize("combo,match", [(dict(), "distribution 'quantile'"),
                                         (dict(distribution="categorical"), "distribution 'quantile'"),
                                         (dict(QR, value_transform="rescale"), "value_transform"),
                                         (dict(QR, augment_m=2), "augment_m"), (dict(QR, augment_k=2), "augment_m"),
                                         (dict(QR, augment_m=2, augment_k=2, quantile_average_copies=True), "augment_m")])
def test_combinations_are_refused_naming_the_switch(combo, match):
    from rainbow_b200.agent import munchausen_options
    with pytest.raises(ValueError, match=match) as e:
        munchausen_options(make_args(munchausen=True, **combo))
    assert "munchausen" in str(e.value)
    assert munchausen_options(make_args(munchausen=False, **combo)) is None


def test_composable_switches_are_accepted():
    from rainbow_b200.agent import munchausen_options
    kw = dict(QR, munchausen=True, augment_shift=4, augment_intensity=0.05, anneal_steps=100, target_tau=0.005,
              reset_interval=10, redo_interval=5, weight_decay=0.1, reset_optimizer=True, learn_stats=8,
              value_transform="none", augment_m=1, augment_k=1)
    assert munchausen_options(make_args(**kw)) is not None


# ---- the C entries -----------------------------------------------------------------------------------------------------------
_CT = {"const float*": ctypes.c_void_p, "float*": ctypes.c_void_p, "const int64_t*": ctypes.c_void_p,
       "int": ctypes.c_int32, "float": ctypes.c_float, "rb_stream_t": ctypes.c_void_p}


def _header_args(name):
    text = open(os.path.join(ROOT, "include", "rainbow_b200.h")).read()
    body = re.search(r"int\s+" + name + r"\s*\(([^)]*)\)", text).group(1)
    return [_CT[re.sub(r"\s*\w+$", "", a.strip()).replace(" *", "*")] for a in body.split(",")]


@pytest.mark.parametrize("name", ["rb_qr_dueling_munchausen_loss_grad", "rb_qr_munchausen_loss_grad"])
def test_signatures_match_the_header(name):
    from rainbow_b200 import _lib
    ret, args = _lib.SIGNATURES[name]
    assert ret is ctypes.c_int
    assert [ctypes.c_void_p if a is ctypes.c_void_p else a for a in args] == _header_args(name)
    assert hasattr(lib(), name)
    assert lib().rb_abi_version() == 3, "additive entries: the ABI version stays"


def test_dueling_refusals_without_gpu():
    # z_online, z_target, A, N, actions, returns, nonterminals, weights, kappa, gamma_n, alpha, temperature, clip, B,
    # loss, dz, theta_out, bonus_out, stream
    good = [ONE, ONE, 6, 51] + [ONE] * 4 + [1.0, 0.97, 0.9, 0.03, -1.0, 32, ONE, ONE, None, None, None]
    fn = lib().rb_qr_dueling_munchausen_loss_grad

    def call(**change):
        a = list(good)
        for i, v in change.items():
            a[int(i[1:])] = v
        return fn(*a)

    for i in (0, 1, 4, 5, 6, 7, 14, 15):
        assert call(**{f"a{i}": None}) == RB_ERR_INVAL, i
        assert b"null" in lib().rb_last_error()
    for i, v in ((13, 0), (13, -3), (2, 0), (3, 1)):
        assert call(**{f"a{i}": v}) == RB_ERR_INVAL, (i, v)
    for k in (0.0, -1.0, math.nan, math.inf):
        assert call(a8=k) == RB_ERR_INVAL and b"kappa" in lib().rb_last_error(), k
    _parameter_refusals(call, 10)
    assert call(a3=129) == RB_ERR_RANGE
    assert call(a2=200, a3=128) == RB_ERR_RANGE and b"too large" in lib().rb_last_error()


def test_plain_refusals_without_gpu():
    # q_online_s, q_target_s, q_target_ns, actions, returns, nonterminals, weights, kappa, gamma_n, alpha, temperature,
    # clip, B, A, N, loss, grad, theta_out, bonus_out, stream
    good = [ONE] * 7 + [1.0, 0.97, 0.9, 0.03, -1.0, 32, 6, 51, ONE, ONE, None, None, None]
    fn = lib().rb_qr_munchausen_loss_grad

    def call(**change):
        a = list(good)
        for i, v in change.items():
            a[int(i[1:])] = v
        return fn(*a)

    for i in (0, 1, 2, 3, 4, 5, 6, 15, 16):
        assert call(**{f"a{i}": None}) == RB_ERR_INVAL, i
        assert b"null" in lib().rb_last_error()
    for k in (0.0, math.nan):
        assert call(a7=k) == RB_ERR_INVAL and b"kappa" in lib().rb_last_error(), k
    _parameter_refusals(call, 9)
    assert call(a14=129) == RB_ERR_RANGE
    assert call(a13=20000) == RB_ERR_RANGE and b"too many actions" in lib().rb_last_error()


def _parameter_refusals(call, ia):
    for a in (-0.1, 1.01, math.nan, math.inf):
        assert call(**{f"a{ia}": a}) == RB_ERR_INVAL and b"alpha" in lib().rb_last_error(), a
    for t in (0.0, -0.03, 1e-40, math.nan, math.inf):
        assert call(**{f"a{ia + 1}": t}) == RB_ERR_INVAL and b"temperature" in lib().rb_last_error(), t
    for c in (0.0, 0.5, math.nan, -math.inf):
        assert call(**{f"a{ia + 2}": c}) == RB_ERR_INVAL and b"clip" in lib().rb_last_error(), c
    for a, t, c in ((0.0, 0.03, -1.0), (1.0, 1.0, -1e-3), (0.9, np.finfo(np.float32).tiny, -1e30)):
        # accepted: validation passes and the call then fails only at the pointers' absence of a device (or launches
        # nothing on a CPU-only host); what matters is that none of the three is refused
        rc = call(**{f"a{ia}": a, f"a{ia + 1}": t, f"a{ia + 2}": c})
        assert not (rc == RB_ERR_INVAL and any(w in lib().rb_last_error() for w in (b"alpha", b"temperature", b"clip")))


# ---- the reference -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,A,N,kappa,tau,alpha", [(14, 6, 51, 1.0, 0.03, 0.9), (7, 1, 2, 0.25, 1.0, 0.9),
                                                   (13, 18, 33, 10.0, 0.03, 0.0), (8, 3, 128, 1.0, 1.0, 0.5)])
def test_reference_is_autograd_of_the_objective(B, A, N, kappa, tau, alpha):
    inp = MR.make_inputs("dueling", B, A, N, kappa, 100 * B + N, alpha=alpha, tau=tau)
    T = MR.targets(inp)[0]
    (loss, _), (g, gs) = MR.loss_grad(inp, T)
    dz, _ = MR.dz(inp, g, gs)
    z = inp["z_on"].double().requires_grad_()
    loss_ag, obj = MR.objective(dict(inp, z_on=z))
    obj.backward()
    assert torch.allclose(loss, loss_ag.detach(), rtol=1e-12, atol=1e-14)
    assert torch.allclose(dz, z.grad, rtol=1e-10, atol=1e-15)
    zero_w = inp["weights"] == 0
    assert bool(zero_w.any()) and bool((dz[zero_w] == 0).all())


def _plain(B, A, N, seed, **kw):
    return MR.make_inputs("plain", B, A, N, 1.0, seed, **kw)


def test_one_action_gives_l_zero_and_the_plain_target():
    inp = _plain(12, 1, 51, 4)
    pi, l, _, _ = MR.policy(Q.means(MR.target_logits(inp, "s")[0], 0.0)[0], inp["tau"])
    assert bool((l == 0).all()) and bool((pi == 1).all())
    T, _, b, _, _ = MR.targets(inp)
    assert bool((b == 0).all())
    sc = Q.nonterminal_scale(inp["nonterminals"], inp["gamma_n"]).unsqueeze(1)
    want = inp["returns"].double().unsqueeze(1) + sc * inp["q_tg_ns"].double()[:, 0]
    assert torch.equal(T, want)


def test_alpha_zero_removes_the_bonus():
    a, z = _plain(21, 6, 51, 5), _plain(21, 6, 51, 5, alpha=0.0)
    Ta, _, ba, _, _ = MR.targets(a)
    Tz, _, bz, _, _ = MR.targets(z)
    assert bool((bz == 0).all()) and bool((ba < 0).any())
    assert torch.allclose(Ta - Tz, ba.unsqueeze(1).expand_as(Ta), rtol=0, atol=1e-12)


def test_small_temperature_approaches_the_target_nets_arg_max():
    """On rows whose target mean quantiles are untied, tau -> 0 gives c_j -> theta_j(s', a*) with a* the target net's
    arg-max (l_a* -> 0), and b -> alpha max(q_a(s) - max q(s), l0)."""
    inp = _plain(21, 6, 51, 6)
    qn, _ = MR.target_logits(inp, "ns")
    qs, _ = MR.target_logits(inp, "s")
    ev_n, ev_s = qn.mean(2), qs.mean(2)
    top2 = ev_n.topk(2, 1).values
    untied = (top2[:, 0] - top2[:, 1]) > 1e-2
    assert int(untied.sum()) >= 10
    best = ev_n.argmax(1)
    sc = Q.nonterminal_scale(inp["nonterminals"], inp["gamma_n"]).unsqueeze(1)
    acts = inp["actions"].long()
    b_lim = inp["alpha"] * torch.clamp_min(C._row(ev_s, acts) - ev_s.max(1).values, inp["clip"])
    want = inp["returns"].double().unsqueeze(1) + b_lim.unsqueeze(1) + sc * C._row(qn, best)
    for tau in (1e-4, 1e-5):
        T, _, b, _, _ = MR.targets(dict(inp, tau=tau))
        assert float((T - want)[untied].abs().max()) < 1e-2 * tau / 1e-4 + 1e-9
    T, _, _, _, _ = MR.targets(dict(inp, tau=1e-5, alpha=0.0))
    qr_T = inp["returns"].double().unsqueeze(1) + sc * C._row(qn, best)
    assert float((T - qr_T)[untied].abs().max()) < 1e-3, "alpha 0: the QR target with the target net's arg-max"


def test_inputs_have_clipped_and_unclipped_rows():
    for tau in (0.03, 1.0):
        inp = _plain(84, 6, 51, 7, tau=tau)
        _, _, b, _, near = MR.targets(inp)
        clipped = b == inp["alpha"] * inp["clip"]
        assert bool(clipped.any()) and bool((~clipped).any()), tau
        assert int(near.sum()) <= 2


@pytest.mark.parametrize("tau,A,N", [(0.03, 6, 51), (1.0, 18, 128), (0.03, 3, 2), (0.003, 6, 51)])
def test_error_scale_covers_an_fp32_emulation(tau, A, N):
    """The derived scale of T against the kernel's operation order in fp32, with the mean quantiles formed in fp32, every
    expf / logf result moved by up to its documented ulps; the largest error stays below TAU x scale, and above a
    twentieth of it on some row (the scale is not loose by orders of magnitude)."""
    rng = np.random.default_rng(11)
    B = 84
    inp = _plain(B, A, N, 17, tau=tau)
    T64, scale, b64, bs, _ = MR.targets(inp)
    worst = 0.0
    for i in range(B):
        qs32 = inp["q_tg_s"][i].numpy()
        qn32 = inp["q_tg_ns"][i].numpy()
        mean32 = lambda q: np.array([np.float32(np.sum(r, dtype=np.float32) / np.float32(N)) for r in q], np.float32)
        act = int(inp["actions"][i])
        sc = np.float32(np.float32(inp["nonterminals"][i, 0]) * np.float32(inp["gamma_n"]))
        T32, b32 = MR.emulate_fp32(mean32(qs32), mean32(qn32), qn32, act, np.float32(inp["returns"][i]), sc,
                                   inp["alpha"], inp["tau"], inp["clip"], rng)
        err = np.abs(T32.astype(np.float64) - T64[i].numpy())
        worst = max(worst, float((err / scale[i].numpy()).max()))
        assert abs(float(b32) - float(b64[i])) <= Q.TAU * float(bs[i])
    assert worst <= Q.TAU, worst
    assert worst >= Q.TAU / 20, f"scale loose: {worst:.3g} of TAU {Q.TAU}"


def test_slips_move_elements_past_the_tolerance():
    """The single-point slips DESIGN.md §17 lists as kernel mutations move some T element by >= 5 x TAU of its scale, so
    the GPU per-element test catches each."""
    inp = _plain(42, 6, 51, 3)
    T, sc, b, _, _ = MR.targets(inp)
    rel = lambda got: float(torch.nan_to_num((got - T).abs() / sc, nan=0.0).max())
    alpha, tau, l0 = inp["alpha"], inp["tau"], inp["clip"]
    qn = MR.target_logits(inp, "ns")[0]
    qs = MR.target_logits(inp, "s")[0]
    pi, l, _, _ = MR.policy(qn.mean(2), tau)
    r = inp["returns"].double().unsqueeze(1)
    s = Q.nonterminal_scale(inp["nonterminals"], inp["gamma_n"]).unsqueeze(1)
    acts = inp["actions"].long()
    c = (pi.unsqueeze(-1) * (qn - l.unsqueeze(-1))).sum(1)
    l_s = MR.policy(qs.mean(2), tau)[1]
    b_ns = alpha * torch.clamp_min(C._row(l, acts), l0)
    slips = {
        "bonus from the s' row": r + b_ns.unsqueeze(1) + s * c,
        "no -l' term": r + b.unsqueeze(1) + s * (pi.unsqueeze(-1) * qn).sum(1),
        "clip dropped": r + alpha * C._row(l_s, acts).unsqueeze(1) + s * c,
        "nt applied to b": r + s * b.unsqueeze(1) + s * c,
        "online rows for pi": r + b.unsqueeze(1) + s * (MR.policy(inp["q_on_s"].double().mean(2), tau)[0].unsqueeze(-1) *
                                                        (qn - MR.policy(inp["q_on_s"].double().mean(2), tau)[1].unsqueeze(-1))).sum(1),
    }
    for name, got in slips.items():
        assert rel(got) >= 5 * Q.TAU, f"{name}: {rel(got):.3g}"
