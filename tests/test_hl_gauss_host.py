"""HL-Gauss targets without a GPU: the options (args.categorical_target, args.hl_gauss_sigma) and every refusal, the two C
entries' signatures against the header and their host-side refusals, and tests/hlg_ref.py -- its masses against an
independent normal-CDF formula, its gradient against autograd, its limits, and the derived error bounds against an fp32
emulation of the stated operation order."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

import c51_ref as C
import hlg_ref as H
from test_qr_host import make_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RB_ERR_INVAL = -22
ONE = 8   # a pointer that is never dereferenced: validation fails first
HLG = dict(categorical_target="hl_gauss")


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


# ---- options ---------------------------------------------------------------------------------------------------------------
def test_defaults_and_off():
    from rainbow_b200.agent import hl_gauss_options
    for off in (dict(), dict(categorical_target=None), dict(categorical_target="projection")):
        assert hl_gauss_options(make_args(**off)) is None
        assert hl_gauss_options(make_args(distribution="quantile", value_transform="rescale", risk_measure="cvar",
                                          augment_m=2, hl_gauss_sigma="x", **off)) is None, "sigma is read only when on"
    assert hl_gauss_options(make_args(**HLG)) == 0.75
    assert hl_gauss_options(make_args(**HLG, hl_gauss_sigma=None)) == 0.75
    assert hl_gauss_options(make_args(**HLG, hl_gauss_sigma=100)) == 100.0
    assert hl_gauss_options(make_args(**HLG, hl_gauss_sigma=np.float32(0.05))) == float(np.float32(0.05))
    assert hl_gauss_options(make_args(**HLG, risk_measure="neutral", value_transform="none")) == 0.75


@pytest.mark.parametrize("bad", ["HL-Gauss", "gauss", 1, True])
def test_unknown_target_is_refused(bad):
    from rainbow_b200.agent import hl_gauss_options
    with pytest.raises(ValueError, match="categorical_target"):
        hl_gauss_options(make_args(categorical_target=bad))


@pytest.mark.parametrize("bad", [0, -1, math.nan, math.inf, 1e-50, 1e3, "0.75", True])
def test_bad_sigma_is_refused(bad):
    from rainbow_b200.agent import hl_gauss_options
    with pytest.raises(ValueError, match="hl_gauss_sigma"):
        hl_gauss_options(make_args(**HLG, hl_gauss_sigma=bad))


@pytest.mark.parametrize("combo,match", [(dict(distribution="quantile"), "distribution"),
                                         (dict(value_transform="rescale"), "value_transform"),
                                         (dict(risk_measure="cvar"), "risk_measure"),
                                         (dict(risk_measure="wang"), "risk_measure"),
                                         (dict(augment_m=2), "augment_m"), (dict(augment_k=2), "augment_m"),
                                         (dict(augment_m=2, augment_k=4), "augment_m")])
def test_combinations_are_refused_naming_the_switch(combo, match):
    from rainbow_b200.agent import hl_gauss_options
    with pytest.raises(ValueError, match=match) as e:
        hl_gauss_options(make_args(**HLG, **combo))
    assert "categorical_target" in str(e.value)


def test_munchausen_keeps_its_own_refusal():
    from rainbow_b200.agent import munchausen_options
    with pytest.raises(ValueError, match="munchausen needs distribution 'quantile'"):
        munchausen_options(make_args(**HLG, munchausen=True))


def test_composable_switches_are_accepted():
    from rainbow_b200.agent import hl_gauss_options
    kw = dict(augment_shift=4, augment_intensity=0.05, anneal_steps=100, target_tau=0.005, reset_interval=10,
              redo_interval=5, weight_decay=0.1, reset_optimizer=True, learn_stats=8, tf32=True, cuda_graph=True,
              fused_head=False, bootstrap_truncation=True, world_size=2, peer_optimizer=True, value_transform="none",
              risk_measure=None, munchausen=False, augment_m=1, augment_k=1, distribution="categorical")
    assert hl_gauss_options(make_args(**HLG, hl_gauss_sigma=2.0, **kw)) == 2.0


# ---- the C entries -----------------------------------------------------------------------------------------------------------
_CT = {"const float*": ctypes.c_void_p, "float*": ctypes.c_void_p, "const int64_t*": ctypes.c_void_p,
       "int64_t*": ctypes.c_void_p, "int": ctypes.c_int32, "float": ctypes.c_float, "rb_stream_t": ctypes.c_void_p}
ENTRIES = {"rb_c51_hlg_loss_grad": "rb_c51_loss_grad", "rb_c51_dueling_hlg_loss_grad": "rb_c51_dueling_loss_grad"}


def _header_args(name):
    text = open(os.path.join(ROOT, "include", "rainbow_b200.h")).read()
    body = re.search(r"int\s+" + name + r"\s*\(([^)]*)\)", text).group(1)
    return [_CT[re.sub(r"\s*\w+$", "", a.strip()).replace(" *", "*")] for a in body.split(",")]


def _header_names(name):
    text = open(os.path.join(ROOT, "include", "rainbow_b200.h")).read()
    body = re.search(r"int\s+" + name + r"\s*\(([^)]*)\)", text).group(1)
    return [re.search(r"(\w+)$", a.strip()).group(1) for a in body.split(",")]


@pytest.mark.parametrize("name", ENTRIES)
def test_signatures_match_the_header(name):
    from rainbow_b200 import _lib
    ret, args = _lib.SIGNATURES[name]
    assert ret is ctypes.c_int
    assert list(args) == _header_args(name)
    names, parent = _header_names(name), _header_names(ENTRIES[name])
    g = parent.index("gamma_n") + 1
    assert names == parent[:g] + ["sigma"] + parent[g:-1] + ["y_out", "stream"], \
        "the parent's arguments, sigma after gamma_n and y_out before the stream"
    assert _header_args(ENTRIES[name]) == [a for i, a in enumerate(_header_args(name)) if names[i] not in ("sigma", "y_out")]
    assert hasattr(lib(), name)
    assert lib().rb_abi_version() == 3, "additive entries: the ABI version stays"


def _good_args(name):
    """Arguments every check accepts, by the entry's header types (pointers ONE, sizes small, sigma 0.3)."""
    names = _header_names(name)
    args = [ONE if t is ctypes.c_void_p else (6 if t is ctypes.c_int32 else 1.0) for t in _header_args(name)]
    args[-1] = None
    args[names.index("sigma")] = 0.3
    return args, names


@pytest.mark.parametrize("name", ENTRIES)
def test_refusals_without_gpu(name):
    fn = getattr(lib(), name)
    good, names = _good_args(name)
    s = names.index("sigma")
    for bad in (math.nan, math.inf, -math.inf, 0.0, -0.0, -1.0, 1e-39, 1e-45):
        a = list(good)
        a[s] = bad
        assert fn(*a) == RB_ERR_INVAL, bad
        msg = lib().rb_last_error().decode()
        assert msg.startswith(name) and "sigma" in msg, msg
    for ptr in [i for i, n in enumerate(names) if n not in ("m_out", "astar_out", "y_out", "stream")
                and _header_args(name)[i] is ctypes.c_void_p]:
        a = list(good)
        a[ptr] = None
        assert fn(*a) == RB_ERR_INVAL, names[ptr]
        assert "null" in lib().rb_last_error().decode()
    # the parent's refusals come first: a null first pointer with a bad sigma is refused as the parent refuses it
    a = list(good)
    a[0], a[s] = None, math.nan
    assert fn(*a) == RB_ERR_INVAL
    assert "null" in lib().rb_last_error().decode()


# ---- the reference -------------------------------------------------------------------------------------------------------------
def _case(Z=51, sup="pm10", ratio=0.75, B=55, seed=3, A=6, entry="plain"):
    inp = H.make_inputs(entry, B, A, Z, sup, seed, ratio)
    ev, _ = C.expected_values(inp)
    return inp, ev.argmax(1)


@pytest.mark.parametrize("ratio", [0.05, 0.1, 0.75, 4.0, 100.0])
@pytest.mark.parametrize("sup", ["pm10", "0to20", "pm100"])
def test_masses_match_the_normal_cdf(ratio, sup):
    inp, astar = _case(sup=sup, ratio=ratio)
    (y, _), (m, _) = H.target(inp, astar)
    sigma = 1.0 / (math.sqrt(2.0) * H.c_of(inp["sigma"]))
    want = H.masses_ndtr(y.numpy(), sigma, H.edges(inp["support"], inp["dz"]).numpy())
    assert np.allclose(m.numpy(), want, rtol=1e-9, atol=1e-15)
    assert torch.allclose(m.sum(1), torch.ones(m.shape[0], dtype=torch.float64), rtol=0, atol=1e-12)


def test_gradient_matches_autograd():
    inp, astar = _case(entry="plain", B=35)
    _, (m, _) = H.target(inp, astar)
    q = C._d(inp["q_on_s"]).clone().requires_grad_(True)
    acts = inp["actions"]
    rows = q[torch.arange(q.shape[0]), acts]
    loss = -(m * torch.log_softmax(rows, -1)).sum(1)
    (lsum,) = torch.autograd.grad((loss * C._d(inp["weights"])).sum() / inp["B"], q)
    (l_ref, _), (g_ref, _) = H.loss_grad(inp, m, torch.zeros_like(m))
    assert torch.allclose(l_ref, loss.detach(), rtol=1e-12, atol=1e-14)
    assert torch.allclose(lsum[torch.arange(q.shape[0]), acts], g_ref, rtol=1e-10, atol=1e-16)


def test_limits():
    inp, astar = _case(ratio=0.75, B=55)
    (y, _), (m, _) = H.target(inp, astar)
    nt, r = inp["nonterminals"].reshape(-1), C._d(inp["returns"])
    term = nt == 0
    assert torch.equal(y[term], r[term].clamp(inp["vmin"], inp["vmax"])), "a terminal row's target is r"
    e = H.edges(inp["support"], inp["dz"])
    # sigma -> 0: all the mass in y's bin, split evenly on an edge
    tiny = dict(inp, sigma=1e-30)
    (y0, _), (m0, _) = H.target(tiny, astar)
    for i in range(inp["B"]):
        k = int(torch.searchsorted(e, y0[i], right=True)) - 1
        on_edge = bool((e == y0[i]).any()) and 0 < k < inp["Z"]
        if on_edge:
            assert float(m0[i, k - 1]) == 0.5 and float(m0[i, k]) == 0.5, i
        else:
            assert float(m0[i, min(k, inp["Z"] - 1)]) == 1.0, i
    assert any(((e == v).any() and v > e[0] and v < e[-1]) for v in y0), "the inputs hold an interior edge row"
    # y at the centre of a symmetric support: a symmetric histogram
    mid = dict(inp, returns=torch.zeros(inp["B"]), nonterminals=torch.zeros(inp["B"], 1))
    _, (ms, ems) = H.target(mid, astar)
    assert bool(((ms - ms.flip(1)).abs() <= ems).all()), "symmetric up to the fp32 support's own asymmetry (1 ulp)"


# ---- the bound against an fp32 emulation -----------------------------------------------------------------------------------
def _perturb(v, ulps, rng):
    """fp32 v moved by a random whole number of its ulps in [-ulps, ulps]."""
    v = v.astype(np.float32)
    k = rng.integers(-ulps, ulps + 1, size=v.shape)
    return (v.astype(np.float64) + k * np.spacing(np.abs(v)).astype(np.float64)).astype(np.float32)


def emulate(inp, astar, rng):
    """(y, m) of the stated fp32 operation order, with erff / erfcf moved by up to their ulps and ybar by up to its bound."""
    from scipy.special import erf, erfc
    f = np.float32
    yb, eyb = H.ybar(inp, astar)
    yb = (yb.numpy() + rng.uniform(-1, 1, yb.shape) * eyb.numpy()).astype(f)
    sc = H.sc_of(inp).numpy().astype(f)
    r = inp["returns"].reshape(-1).numpy().astype(f)
    y = np.clip((r + (sc * yb).astype(f)).astype(f), f(inp["vmin"]), f(inp["vmax"]))
    c = f(H.c_of(inp["sigma"]))
    e = H.edges(inp["support"], inp["dz"]).numpy().astype(f)
    t = ((e[None, :] - y[:, None]).astype(f) * c).astype(f)
    t0, t1 = t[:, :-1], t[:, 1:]

    def fn(g, x, ulps):
        return _perturb(g(x.astype(np.float64)).astype(f), ulps, rng)
    d = np.where(t0 >= 0, fn(erfc, t0, H.ERFC_ULP) - fn(erfc, t1, H.ERFC_ULP),
                 np.where(t1 <= 0, fn(erfc, -t1, H.ERFC_ULP) - fn(erfc, -t0, H.ERFC_ULP),
                          fn(erf, t1, H.ERF_ULP) - fn(erf, t0, H.ERF_ULP))).astype(f)
    u = (f(0.5) * d).astype(f)
    B, Z = u.shape
    lanes = np.zeros((B, 32), f)
    for k in range(Z):                       # each lane over its atoms k = lane + 32 r in r order
        lanes[:, k % 32] = (lanes[:, k % 32] + u[:, k]).astype(f)
    for o in (16, 8, 4, 2, 1):               # the xor butterfly
        lanes = (lanes + lanes[:, np.arange(32) ^ o]).astype(f)
    return y, (u / lanes[:, :1]).astype(f)


@pytest.mark.parametrize("ratio", [0.05, 0.1, 0.75, 4.0, 100.0])
@pytest.mark.parametrize("Z,sup", [(2, "pm10"), (51, "pm10"), (101, "0to20"), (51, "pm100"), (128, "pm1")])
def test_fp32_emulation_is_within_the_bound(ratio, Z, sup):
    rng = np.random.default_rng(Z * 1000 + int(ratio * 100))
    inp, astar = _case(Z=Z, sup=sup, ratio=ratio, B=55, seed=Z)
    assert {C.RET_KINDS[i % 5] for i in range(inp["B"])} == set(C.RET_KINDS)
    (y, ey), (m, em) = H.target(inp, astar)
    worst_y = worst_m = 0.0
    for _ in range(4):
        ye, me = emulate(inp, astar, rng)
        dy = np.abs(ye.astype(np.float64) - y.numpy())
        dm = np.abs(me.astype(np.float64) - m.numpy())
        assert (dy <= ey.numpy()).all(), (dy / ey.numpy()).max()
        assert (dm <= em.numpy()).all(), (dm / em.numpy()).max()
        worst_y, worst_m = max(worst_y, (dy / ey.numpy()).max()), max(worst_m, (dm / em.numpy()).max())
    # the loss and gradient bounds of the emulated m hold against the reference's
    (l_ref, el), (g_ref, eg) = H.loss_grad(inp, m, em)
    (l_e, _), (g_e, _) = C.loss_grad(inp, torch.from_numpy(me.astype(np.float64)))
    assert bool(((l_e - l_ref).abs() <= el).all()) and bool(((g_e - g_ref).abs() <= eg).all())


@pytest.mark.parametrize("ratio", [0.1, 0.75, 4.0])
def test_bound_sees_the_slips(ratio):
    """Each slip the kernel could make in the definition moves m far past the bound: edges at the atoms, no
    normalisation, sigma not scaled by dz."""
    inp, astar = _case(ratio=ratio, sup="pm100", B=55)
    (y, _), (m, em) = H.target(inp, astar)
    sup = C._d(inp["support"])
    c = H.c_of(inp["sigma"])

    def masses(e, cc, norm=True):
        t = (e.unsqueeze(0) - y.unsqueeze(1)) * cc
        u = 0.5 * (torch.erf(t[:, 1:]) - torch.erf(t[:, :-1]))
        return u / u.sum(1, keepdim=True) if norm else u
    e = H.edges(inp["support"], inp["dz"])
    at_atoms = torch.cat([sup, sup[-1:] + inp["dz"]])
    for name, got in (("edges at the atoms", masses(at_atoms, c)), ("no normalisation", masses(e, c, norm=False)),
                      ("sigma not scaled", masses(e, H.c_of(C.f32(ratio))))):
        assert ((got - m).abs() / em).max() > 10, name
