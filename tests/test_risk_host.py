"""Risk-sensitive selection without a GPU: the options (args.risk_measure, args.risk_eta) and every refusal, the six C
entries' signatures against the header and their host-side refusals, and tests/risk_ref.py -- beta against the standard
library, the limits (CVaR at eta = 1 and Wang at eta = 0 are the mean, CVaR as eta -> 0 the lowest atom or theta_0), the
telescoping weights, the torch fallback of Agent.q_select, and the derived bound against an fp32 emulation of the stated
operation order."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

import c51_ref as C
import qr_ref as Q
import risk_ref as RR
from test_qr_host import make_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RB_ERR_INVAL = -22
ONE = 8   # a pointer that is never dereferenced: validation fails first
QR = dict(distribution="quantile")
MEASURES = [("cvar", 0.1), ("cvar", 0.25), ("cvar", 1.0), ("wang", -0.75), ("wang", 0.0), ("wang", 0.75)]


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


# ---- options ---------------------------------------------------------------------------------------------------------------
def test_defaults_and_off():
    from rainbow_b200.agent import risk_options
    for off in (dict(), dict(risk_measure=None), dict(risk_measure="neutral")):
        assert risk_options(make_args(**off)) is None
        assert risk_options(make_args(**QR, **off)) is None
        assert risk_options(make_args(value_transform="rescale", munchausen=True, augment_m=2, risk_eta="x", **off)) is None
    assert risk_options(make_args(risk_measure="cvar")) == ("cvar", 0.25)
    assert risk_options(make_args(risk_measure="wang", **QR)) == ("wang", -0.75)
    assert risk_options(make_args(risk_measure="cvar", risk_eta=None)) == ("cvar", 0.25)
    assert risk_options(make_args(risk_measure="cvar", risk_eta=1)) == ("cvar", 1.0)
    assert risk_options(make_args(risk_measure="wang", risk_eta=0.1)) == ("wang", float(np.float32(0.1))), \
        "eta is rounded to the fp32 the kernels take"
    assert risk_options(make_args(risk_measure="wang", risk_eta=0)) == ("wang", 0.0)


@pytest.mark.parametrize("measure,bad", [("cvar", v) for v in (0.0, -0.25, 1.5, math.nan, math.inf, 1e-50, "0.5", True)] +
                         [("wang", v) for v in (math.nan, math.inf, -math.inf, 1e39, -1e39, "x", False)])
def test_bad_eta_is_refused(measure, bad):
    from rainbow_b200.agent import risk_options
    with pytest.raises(ValueError, match="risk_eta"):
        risk_options(make_args(risk_measure=measure, risk_eta=bad))


@pytest.mark.parametrize("bad", ["CVaR", "pow", "cpw", 1, True])
def test_unknown_measure_is_refused(bad):
    from rainbow_b200.agent import risk_options
    with pytest.raises(ValueError, match="risk_measure"):
        risk_options(make_args(risk_measure=bad))


@pytest.mark.parametrize("combo,match", [(dict(value_transform="rescale"), "value_transform"),
                                         (dict(QR, value_transform="rescale"), "value_transform"),
                                         (dict(QR, munchausen=True), "munchausen"),
                                         (dict(augment_m=2), "augment_m"), (dict(augment_k=2), "augment_m"),
                                         (dict(QR, augment_m=2, augment_k=2, quantile_average_copies=True), "augment_m")])
def test_combinations_are_refused_naming_the_switch(combo, match):
    from rainbow_b200.agent import risk_options
    for measure in ("cvar", "wang"):
        with pytest.raises(ValueError, match=match) as e:
            risk_options(make_args(risk_measure=measure, **combo))
        assert "risk_measure" in str(e.value)


def test_composable_switches_are_accepted():
    from rainbow_b200.agent import risk_options
    kw = dict(augment_shift=4, augment_intensity=0.05, anneal_steps=100, target_tau=0.005, reset_interval=10,
              redo_interval=5, weight_decay=0.1, reset_optimizer=True, learn_stats=8, value_transform="none",
              munchausen=False, augment_m=1, augment_k=1)
    for dist in (dict(), QR):
        assert risk_options(make_args(risk_measure="cvar", **dist, **kw)) == ("cvar", 0.25)


# ---- the C entries -----------------------------------------------------------------------------------------------------------
_CT = {"const float*": ctypes.c_void_p, "float*": ctypes.c_void_p, "const int64_t*": ctypes.c_void_p,
       "int64_t*": ctypes.c_void_p, "int": ctypes.c_int32, "float": ctypes.c_float, "rb_stream_t": ctypes.c_void_p}
ENTRIES = ["rb_c51_risk_loss_grad", "rb_c51_dueling_risk_loss_grad", "rb_qr_dueling_risk_loss_grad", "rb_qr_risk_loss_grad",
           "rb_q_values_risk", "rb_qr_q_values_risk"]


def _header_args(name):
    text = open(os.path.join(ROOT, "include", "rainbow_b200.h")).read()
    body = re.search(r"int\s+" + name + r"\s*\(([^)]*)\)", text).group(1)
    return [_CT[re.sub(r"\s*\w+$", "", a.strip()).replace(" *", "*")] for a in body.split(",")]


@pytest.mark.parametrize("name", ENTRIES)
def test_signatures_match_the_header(name):
    from rainbow_b200 import _lib
    ret, args = _lib.SIGNATURES[name]
    assert ret is ctypes.c_int
    assert [ctypes.c_void_p if a is ctypes.c_void_p else a for a in args] == _header_args(name)
    parent = _lib.SIGNATURES[name.replace("_risk", "")][1]
    assert list(args) == list(parent[:-1]) + [ctypes.c_int, ctypes.c_float, parent[-1]], \
        "the parent's arguments, then risk_kind and risk_eta before the stream"
    assert hasattr(lib(), name)
    assert lib().rb_abi_version() == 3, "additive entries: the ABI version stays"
    text = open(os.path.join(ROOT, "include", "rainbow_b200.h")).read()
    assert re.search(r"#define RB_RISK_CVAR 1\b", text) and re.search(r"#define RB_RISK_WANG 2\b", text)


def _good_args(name):
    """Arguments every check accepts, by the entry's header types (pointers ONE, sizes small, kappa 1)."""
    args = []
    for t in _header_args(name):
        args.append(ONE if t is ctypes.c_void_p else (6 if t is ctypes.c_int32 else 1.0))
    args[-1] = None                                            # the stream
    args[-3], args[-2] = 1, 0.25                               # CVaR at 0.25
    return args


@pytest.mark.parametrize("name", ENTRIES)
def test_risk_refusals_without_gpu(name):
    fn = getattr(lib(), name)
    good = _good_args(name)
    for kind, eta, what in ((0, 0.25, "risk_kind"), (3, 0.25, "risk_kind"), (-1, 0.0, "risk_kind"),
                            (1, 0.0, "CVaR eta"), (1, -0.5, "CVaR eta"), (1, 1.5, "CVaR eta"), (1, math.nan, "CVaR eta"),
                            (1, math.inf, "CVaR eta"), (2, math.nan, "Wang eta"), (2, math.inf, "Wang eta"),
                            (2, -math.inf, "Wang eta")):
        a = list(good)
        a[-3], a[-2] = kind, eta
        assert fn(*a) == RB_ERR_INVAL, (kind, eta)
        msg = lib().rb_last_error().decode()
        assert msg.startswith(name) and what in msg, msg
    # the parent's refusals come first: a NULL first pointer with a bad kind is refused as the parent refuses it
    a = list(good)
    a[0], a[-3] = None, 7
    assert fn(*a) == RB_ERR_INVAL
    assert "null" in lib().rb_last_error().decode()


# ---- the reference -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("measure,eta", MEASURES)
def test_beta_matches_the_standard_library(measure, eta):
    t = torch.cat([torch.linspace(0, 1, 1001, dtype=torch.float64),
                   torch.tensor([1e-30, 1e-12, 1e-6, 1 - 1e-6, 1 - 1e-9, 1 - 2.0 ** -24], dtype=torch.float64)])
    got = RR.beta(t, measure, eta)
    want = torch.tensor([RR.beta_stdlib(float(v), measure, eta) for v in t], dtype=torch.float64)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-15)
    assert float(got[0]) == 0.0 and float(got[1000]) == 1.0, "beta(0) = 0 and beta(1) = 1 exactly"
    assert bool((got[1:1001] >= got[:1000]).all()), "beta is non-decreasing"


def _rows(seed, M, A, Z, scale=2.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(M, A, Z, generator=g, dtype=torch.float64) * scale


@pytest.mark.parametrize("Z", [2, 51, 128])
def test_neutral_limits_are_the_mean(Z):
    x = _rows(1, 8, 3, Z)
    L = torch.zeros_like(x)
    sup = torch.linspace(-10, 10, Z)
    mean_q = x.mean(-1)
    mean_c = (torch.softmax(x, -1) * sup.double()).sum(-1)
    for measure, eta in (("cvar", 1.0), ("wang", 0.0)):
        Qq, eq = RR.quantile_values(x, L, measure, eta)
        assert bool(((Qq - mean_q).abs() <= eq).all()), measure
        Qc, ec = RR.categorical_values(x, L, sup, measure, eta)
        assert bool(((Qc - mean_c).abs() <= ec).all()), measure
        assert bool((eq < 1e-3).all()) and bool((ec < 1e-3).all()), "the bound stays small at the mean"


def test_cvar_to_zero_is_the_lowest_level():
    x = _rows(2, 4, 3, 51)
    sup = torch.linspace(-10, 10, 51)
    Qq, _ = RR.quantile_values(x, torch.zeros_like(x), "cvar", 1e-6)
    assert torch.allclose(Qq, x[..., 0], rtol=0, atol=1e-12), "CVaR below 1/N is theta_0"
    logits = x.clone()
    logits[..., :3] = -1e4                                     # atoms 0..2 carry no mass (in float64)
    Qc, _ = RR.categorical_values(logits, torch.zeros_like(x), sup, "cvar", 1e-30)
    assert torch.allclose(Qc, torch.full_like(Qc, float(sup[3])), rtol=0, atol=1e-6), "the lowest atom with mass"
    Qw, _ = RR.quantile_values(x, torch.zeros_like(x), "wang", -40.0)
    assert torch.allclose(Qw, x[..., 0], rtol=0, atol=1e-9), "Wang at eta -> -inf is theta_0"


@pytest.mark.parametrize("measure,eta", MEASURES)
def test_weights_telescope_to_one(measure, eta):
    for n in (2, 51, 128):
        b = RR.beta(torch.arange(n + 1, dtype=torch.float64) / n, measure, eta)
        w = b[1:] - b[:-1]
        assert abs(float(w.sum()) - 1.0) < 1e-14 and bool((w >= 0).all())
    x = _rows(3, 5, 2, 51)
    F = torch.softmax(x, -1).cumsum(-1).clamp(max=1)
    F[..., -1] = 1
    b = RR.beta(F, measure, eta)
    w = b - torch.nn.functional.pad(b[..., :-1], (1, 0))
    assert torch.allclose(w.sum(-1), torch.ones(5, 2, dtype=torch.float64), atol=1e-14)


def test_risk_and_mean_disagree_on_the_constructed_rows():
    """Action 0: the higher mean and a heavy lower tail; action 1: a narrow distribution a little below it."""
    N = 51
    a0 = torch.cat([torch.full((5,), -20.0), torch.full((N - 5,), 6.0)]).double()
    a1 = torch.full((N,), 1.5, dtype=torch.float64)
    x = torch.stack([a0, a1]).unsqueeze(0)
    assert float(x[0, 0].mean()) > float(x[0, 1].mean()) + 0.5
    Q_, err = RR.quantile_values(x, torch.zeros_like(x), "cvar", 0.25)
    assert float(Q_[0, 1] - Q_[0, 0]) > 1.0 and float(err.max()) < 1e-3


def test_torch_fallback_matches_the_reference():
    from rainbow_b200.agent import risk_values
    x = _rows(4, 6, 3, 51).float()
    sup = torch.linspace(-10, 10, 51)
    for measure, eta in MEASURES:
        got = risk_values(x, measure, eta)
        want, err = RR.quantile_values(x.double(), torch.zeros_like(x.double()), measure, eta)
        assert bool(((got.double() - want).abs() <= err + 1e-5).all()), measure
        p = torch.softmax(x, -1)
        got = risk_values(p, measure, eta, support=sup)
        want, err = RR.categorical_values(x.double(), torch.zeros_like(x.double()), sup, measure, eta)
        assert bool(((got.double() - want).abs() <= err + 1e-5).all()), measure


@pytest.mark.parametrize("measure,eta", MEASURES)
@pytest.mark.parametrize("Z", [2, 31, 51, 65, 128])
def test_fp32_emulation_is_within_the_bound(measure, eta, Z):
    """The stated operation order in fp32 (torch's CPU exp / ndtr / ndtri standing in for the device functions) against
    the float64 reference, over N(0, 2), sharp N(0, 30) and constant rows; the worst error stays a fraction of the
    bound."""
    worst = 0.0
    for kind, scale in (("n2", 2.0), ("sharp", 30.0), ("const", 0.0)):
        x = _rows(7 + Z, 16, 3, Z, scale if scale else 1.0)
        if kind == "const":
            x = x[..., :1].expand_as(x).contiguous()
        x32 = x.float()
        L = torch.zeros_like(x)
        sup = torch.linspace(-10, 10, Z)
        got = RR.emulate_quantile(x32, measure, eta).double()
        want, err = RR.quantile_values(x32.double(), L, measure, eta)
        assert bool(((got - want).abs() <= err).all()), ("quantile", kind)
        worst = max(worst, float(((got - want).abs() / err).max()))
        got = RR.emulate_categorical(x32, sup, measure, eta).double()
        want, err = RR.categorical_values(x32.double(), L, sup, measure, eta)
        assert bool(((got - want).abs() <= err).all()), ("categorical", kind)
        worst = max(worst, float(((got - want).abs() / err).max()))
    assert worst < 0.5, f"the bound is not tight enough to matter: worst error / bound {worst:.3g}"


def test_bound_sees_the_steep_wang_tail():
    """Wang at eta < 0 near F = 1: beta' = exp(eta z - eta^2 / 2) grows without bound for eta > 0 and shrinks for eta < 0
    there; near F = 0 it is the other way round.  The bound follows the slope."""
    t = torch.tensor([0.5, 1 - 1e-4, 1 - 1e-6], dtype=torch.float64)
    dt = torch.full_like(t, 1e-7)
    e = RR.beta_error(t, dt, "wang", 0.75)
    assert float(e[1]) > float(e[0]) and float(e[2]) > 4 * float(e[0])
    e = RR.beta_error(1 - t, dt, "wang", -0.75)
    assert float(e[1]) > float(e[0]) and float(e[2]) > 4 * float(e[0])
    ec = RR.beta_error(t, dt, "cvar", 0.25)
    assert float(ec[2]) <= RR.U, "CVaR is flat at 1 there"
