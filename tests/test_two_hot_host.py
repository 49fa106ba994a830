"""Two-hot targets without a GPU: the options (args.categorical_target = "two_hot") and every refusal, the four C entries'
signatures against the header and their parents' and their host-side refusals, and tests/twohot_ref.py -- its split's
properties, its agreement with c51_ref's projection of a point mass, and the derived error bounds against an fp32 emulation
of the stated operation order."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

import c51_ref as C
import twohot_ref as T
import vt_ref as V
from test_qr_host import make_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RB_ERR_INVAL = -22
ONE = 8   # a pointer that is never dereferenced: validation fails first
TH = dict(categorical_target="two_hot")


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


# ---- options ---------------------------------------------------------------------------------------------------------------
def test_defaults_and_off():
    from rainbow_b200.agent import hl_gauss_options, two_hot_options
    for off in (dict(), dict(categorical_target=None), dict(categorical_target="projection"),
                dict(categorical_target="hl_gauss")):
        assert two_hot_options(make_args(**off)) is False
    assert two_hot_options(make_args(**TH)) is True
    assert two_hot_options(make_args(**TH, value_transform="rescale")) is True, "value rescaling composes"
    assert two_hot_options(make_args(**TH, hl_gauss_sigma="not read")) is True
    assert two_hot_options(make_args(**TH, risk_measure="neutral", value_transform="none")) is True
    assert hl_gauss_options(make_args(**TH)) is None
    assert hl_gauss_options(make_args(**TH, value_transform="rescale", hl_gauss_sigma="x")) is None


@pytest.mark.parametrize("combo,match", [(dict(distribution="quantile"), "distribution"),
                                         (dict(risk_measure="cvar"), "risk_measure"),
                                         (dict(risk_measure="wang"), "risk_measure"),
                                         (dict(augment_m=2), "augment_m"), (dict(augment_k=2), "augment_m"),
                                         (dict(augment_m=2, augment_k=4), "augment_m")])
def test_combinations_are_refused_naming_the_switch(combo, match):
    from rainbow_b200.agent import two_hot_options
    with pytest.raises(ValueError, match=match) as e:
        two_hot_options(make_args(**TH, **combo))
    assert "categorical_target 'two_hot'" in str(e.value)


def test_munchausen_keeps_its_own_refusal():
    from rainbow_b200.agent import munchausen_options
    with pytest.raises(ValueError, match="munchausen needs distribution 'quantile'"):
        munchausen_options(make_args(**TH, munchausen=True))


def test_composable_switches_are_accepted():
    from rainbow_b200.agent import hl_gauss_options, two_hot_options, value_transform_options
    kw = dict(augment_shift=4, augment_intensity=0.05, anneal_steps=100, target_tau=0.005, reset_interval=10,
              redo_interval=5, weight_decay=0.1, reset_optimizer=True, learn_stats=8, tf32=True, cuda_graph=True,
              fused_head=False, bootstrap_truncation=True, world_size=2, peer_optimizer=True, value_transform="rescale",
              risk_measure=None, munchausen=False, augment_m=1, augment_k=1, distribution="categorical")
    args = make_args(**TH, **kw)
    assert two_hot_options(args) is True and hl_gauss_options(args) is None
    assert value_transform_options(args)[0] == "rescale"


# ---- the C entries -----------------------------------------------------------------------------------------------------------
_CT = {"const float*": ctypes.c_void_p, "float*": ctypes.c_void_p, "const int64_t*": ctypes.c_void_p,
       "int64_t*": ctypes.c_void_p, "int": ctypes.c_int32, "float": ctypes.c_float, "rb_stream_t": ctypes.c_void_p}
ENTRIES = {"rb_c51_twohot_loss_grad": "rb_c51_loss_grad", "rb_c51_dueling_twohot_loss_grad": "rb_c51_dueling_loss_grad",
           "rb_c51_twohot_vt_loss_grad": "rb_c51_loss_grad",
           "rb_c51_dueling_twohot_vt_loss_grad": "rb_c51_dueling_loss_grad"}


def _header_decl(name):
    text = open(os.path.join(ROOT, "include", "rainbow_b200.h")).read()
    return re.search(r"int\s+" + name + r"\s*\(([^)]*)\)", text).group(1).split(",")


def _header_args(name):
    return [_CT[re.sub(r"\s*\w+$", "", a.strip()).replace(" *", "*")] for a in _header_decl(name)]


def _header_names(name):
    return [re.search(r"(\w+)$", a.strip()).group(1) for a in _header_decl(name)]


@pytest.mark.parametrize("name", ENTRIES)
def test_signatures_match_the_header_and_the_parent(name):
    from rainbow_b200 import _lib
    ret, args = _lib.SIGNATURES[name]
    assert ret is ctypes.c_int
    assert list(args) == _header_args(name)
    names, parent = _header_names(name), _header_names(ENTRIES[name])
    tail = ["y_out", "support_q", "eps", "stream"] if "_vt_" in name else ["y_out", "stream"]
    assert names == parent[:-1] + tail, "the parent's arguments, then y_out (and support_q, eps) before the stream"
    ptypes = _header_args(ENTRIES[name])
    assert _header_args(name) == ptypes[:-1] + [ctypes.c_void_p] * (2 if "_vt_" in name else 1) + \
        ([ctypes.c_float] if "_vt_" in name else []) + [ctypes.c_void_p]
    if "_vt_" in name:   # the same tail as the parent's own _vt twin
        vt_parent = ENTRIES[name].replace("_loss_grad", "_vt_loss_grad")
        assert _header_names(vt_parent)[-3:] == ["support_q", "eps", "stream"]
    assert hasattr(lib(), name)
    assert lib().rb_abi_version() == 3, "additive entries: the ABI version stays"


def _good_args(name, Z=51):
    """Arguments every check accepts, by the entry's header types (pointers ONE, sizes small, eps 1e-3)."""
    names = _header_names(name)
    args = [ONE if t is ctypes.c_void_p else (6 if t is ctypes.c_int32 else 1.0) for t in _header_args(name)]
    args[-1] = None
    for n in ("Z", "atoms"):
        if n in names:
            args[names.index(n)] = Z
    if "eps" in names:
        args[names.index("eps")] = 1e-3
    return args, names


@pytest.mark.parametrize("name", ENTRIES)
def test_refusals_without_gpu(name):
    fn = getattr(lib(), name)
    good, names = _good_args(name)
    parent = getattr(lib(), ENTRIES[name])
    pgood, pnames = _good_args(ENTRIES[name])
    for ptr in [i for i, n in enumerate(names) if n not in ("m_out", "astar_out", "y_out", "stream")
                and _header_args(name)[i] is ctypes.c_void_p]:
        a = list(good)
        a[ptr] = None
        assert fn(*a) == RB_ERR_INVAL, names[ptr]
        msg = lib().rb_last_error().decode()
        assert msg.startswith(name) and "null" in msg, msg
    # the parent's shape refusals, with the parent's codes
    for field, bad in (("B", 0), ("B", -1), ("A" if "A" in names else "actions_n", 0), ("Z" if "Z" in names else "atoms", 1),
                       ("Z" if "Z" in names else "atoms", 129)):
        a, p = list(good), list(pgood)
        a[names.index(field)], p[pnames.index(field)] = bad, bad
        assert fn(*a) == parent(*p) != 0, (field, bad)
    if "dueling" in name:   # the fused loss's shared-memory limit
        a, p = list(good), list(pgood)
        a[names.index("actions_n")], p[pnames.index("actions_n")] = 4096, 4096
        a[names.index("atoms")], p[pnames.index("atoms")] = 128, 128
        assert fn(*a) == parent(*p) != 0
    if "_vt_" in name:
        e = names.index("eps")
        for bad in (-1e-3, math.nan, 1.5, math.inf):
            a = list(good)
            a[e] = bad
            assert fn(*a) == RB_ERR_INVAL, bad
            assert "eps" in lib().rb_last_error().decode()
        # rb_c51_vt_loss_grad's refusals come first: a bad eps with a null first pointer is refused for eps
        a = list(good)
        a[0], a[e] = None, math.nan
        assert fn(*a) == RB_ERR_INVAL and "eps" in lib().rb_last_error().decode()


# ---- the reference -------------------------------------------------------------------------------------------------------------
def _case(Z=51, sup="pm10", B=55, seed=3, A=6, entry="plain", eps=None):
    inp = T.make_inputs(entry, B, A, Z, sup, seed, eps)
    ev, _ = T.expected_values(inp)
    return inp, ev.argmax(1)


@pytest.mark.parametrize("eps", [None, 1e-3, 0.0])
@pytest.mark.parametrize("Z,sup", [(2, "pm10"), (51, "pm10"), (101, "0to20"), (51, "pm100"), (128, "pm1")])
def test_split_properties(Z, sup, eps):
    inp, astar = _case(Z=Z, sup=sup, eps=eps)
    (y, _), (m, _) = T.target(inp, astar)
    s = C._d(torch.tensor([C.f32(v) for v in inp["support"]]))
    vmin, dz = C.f32(inp["vmin"]), C.f32(inp["dz"])
    nz = m != 0
    assert bool((nz.sum(1) <= 2).all()), "at most two non-zeros"
    first = nz.float().argmax(1)
    last = Z - 1 - nz.flip(1).float().argmax(1)
    assert bool((last - first <= 1).all()), "and adjacent"
    assert bool((m >= 0).all())
    full = (y - vmin) / dz <= Z - 1             # b inside the support: nothing dropped
    assert torch.allclose(m.sum(1)[full], torch.ones(int(full.sum()), dtype=torch.float64), rtol=0, atol=1e-12)
    grid = vmin + dz * torch.arange(Z, dtype=torch.float64)     # the atoms the split sees: Vmin + k dz
    assert torch.allclose((m * grid).sum(1)[full], y[full], rtol=0, atol=1e-9 * (1 + y.abs().max()))
    # the hat form: m_k = max(0, 1 - |k - b|)
    b = (y - vmin) / dz
    hat = (1 - (torch.arange(Z, dtype=torch.float64).unsqueeze(0) - b.unsqueeze(1)).abs()).clamp(min=0)
    assert torch.allclose(m, hat, rtol=0, atol=1e-12)
    # terminal rows give y = r (h(r) under the transform), clamped
    term = inp["nonterminals"].reshape(-1) == 0
    r = C._d(inp["returns"])
    want = (V.h(r, eps) if eps is not None else r).clamp(vmin, C.f32(inp["vmax"]))
    assert torch.allclose(y[term], want[term], rtol=1e-15, atol=0)
    assert s.shape[0] == Z


@pytest.mark.parametrize("Z", [2, 3, 51, 101, 128])
def test_one_hot_at_every_atom(Z):
    vmin, vmax, dz = -10.0, 10.0, 20.0 / (Z - 1)
    k = torch.arange(Z, dtype=torch.float64)
    y = torch.cat([vmin + k * dz, torch.tensor([vmin, vmax])])      # every atom, then Vmin and Vmax once more
    m, _ = T.split(y, vmin, dz, Z)
    assert torch.allclose(m[:Z], torch.eye(Z, dtype=torch.float64), rtol=0, atol=1e-12), "a y on an atom: a one-hot"
    assert float(m[Z, 0]) == 1.0 and float(m[Z + 1, Z - 1]) == pytest.approx(1.0, abs=1e-12)
    b = torch.arange(Z, dtype=torch.float64)          # b exactly an integer: exactly a one-hot, by the fix-ups at the ends
    assert torch.equal(T.split(vmin + b, vmin, 1.0, Z)[0], torch.eye(Z, dtype=torch.float64))
    # clamped targets: the reference clamps before the split
    inp, astar = _case(Z=max(Z, 2), sup="pm10", B=33)
    (yc, _), (mc, _) = T.target(inp, astar)
    for i in range(inp["B"]):
        if i % 11 == 9:
            assert float(yc[i]) == C.f32(inp["vmin"]) and float(mc[i, 0]) == 1.0
        if i % 11 == 10:
            # b = (Vmax - Vmin) / fl32(dz) is Z - 1 only to dz's rounding: what lies past Z - 1 is dropped
            assert float(yc[i]) == C.f32(inp["vmax"]) and float(mc[i, -1]) == pytest.approx(1.0, abs=Z * 2.0 ** -23)


@pytest.mark.parametrize("eps", [None, 1e-3])
@pytest.mark.parametrize("Z,sup", [(51, "pm10"), (101, "0to20"), (2, "pm100"), (62, "pm1")])
def test_split_is_the_projection_of_a_point_mass(Z, sup, eps):
    """c51_ref's projection (vt_ref's under the transform) of a target row that is a point mass on atom j equals the
    split of y = the projected atom's target: a one-hot row's expected value is s_j (s~_j)."""
    inp, astar = _case(Z=Z, sup=sup, B=44, eps=eps)
    B, A = inp["B"], inp["A"]
    g = torch.Generator().manual_seed(Z)
    j = torch.randint(0, Z, (B,), generator=g)
    q = torch.full((B, A, Z), -1e4)
    q[torch.arange(B).unsqueeze(1), torch.arange(A).unsqueeze(0), j.unsqueeze(1)] = 0.0
    inp = dict(inp, q_tg_ns=q)
    (_, _), (m, _) = T.target(inp, astar)
    proj = V.c51_projection(inp, astar) if eps is not None else C.projection(inp, astar)
    assert torch.allclose(m, proj[0], rtol=0, atol=1e-9)


# ---- the bound against an fp32 emulation -----------------------------------------------------------------------------------
def emulate(inp, astar, rng):
    """(y, m) of the stated fp32 operation order, with ybar moved by up to its bound."""
    f = np.float32
    Z = inp["Z"]
    yb, eyb = T.ybar(inp, astar)
    yb = (yb.numpy() + rng.uniform(-1, 1, yb.shape) * eyb.numpy()).astype(f)
    sc = T.H.sc_of(inp).numpy().astype(f)
    r = inp["returns"].reshape(-1).numpy().astype(f)
    x = (r + (sc * yb).astype(f)).astype(f)
    if "eps" in inp:
        x = V.h32(x, inp["eps"]).astype(f)
    vmin, vmax, dz = f(inp["vmin"]), f(inp["vmax"]), f(inp["dz"])
    y = np.clip(x, vmin, vmax).astype(f)
    b = ((y - vmin).astype(f) / dz).astype(f)
    lo, up = np.floor(b).astype(np.int64), np.ceil(b).astype(np.int64)
    lo = np.where((up > 0) & (lo == up), lo - 1, lo)
    up = np.where((lo < Z - 1) & (lo == up), up + 1, up)
    m = np.zeros((b.shape[0], Z + 1), f)
    rows = np.arange(b.shape[0])
    m[rows, lo] = (up.astype(f) - b).astype(f)
    m[rows, up] = (b - lo.astype(f)).astype(f)
    return y, m[:, :Z]


@pytest.mark.parametrize("eps", [None, 1e-3, 0.0])
@pytest.mark.parametrize("Z,sup", [(2, "pm10"), (51, "pm10"), (101, "0to20"), (51, "pm100"), (128, "pm1"),
                                   (100, "pm100"), (62, "pm1")])
def test_fp32_emulation_is_within_the_bound(Z, sup, eps):
    rng = np.random.default_rng(Z * 1000 + (0 if eps is None else 7))
    inp, astar = _case(Z=Z, sup=sup, B=66, seed=Z, eps=eps)
    (y, ey), (m, em) = T.target(inp, astar)
    for _ in range(4):
        ye, me = emulate(inp, astar, rng)
        dy = np.abs(ye.astype(np.float64) - y.numpy())
        dm = np.abs(me.astype(np.float64) - m.numpy())
        assert (dy <= ey.numpy()).all(), (dy / ey.numpy()).max()
        assert (dm <= em.numpy()).all(), (dm / em.numpy()).max()
    (l_ref, el), (g_ref, eg) = T.loss_grad(inp, m, em)
    (l_e, _), (g_e, _) = C.loss_grad(inp, torch.from_numpy(me.astype(np.float64)))
    assert bool(((l_e - l_ref).abs() <= el).all()) and bool(((g_e - g_ref).abs() <= eg).all())


@pytest.mark.parametrize("eps", [None, 1e-3])
def test_bound_sees_the_slips(eps):
    """Each slip the kernel could make in the definition moves m far past the bound on some row: the fix-ups dropped,
    m_l and m_u swapped, no clamp, and under the transform h not applied to y."""
    inp, astar = _case(Z=51, sup="pm10", B=66, eps=eps)
    (y, _), (m, em) = T.target(inp, astar)
    vmin, vmax, dz, Z = C.f32(inp["vmin"]), C.f32(inp["vmax"]), C.f32(inp["dz"]), inp["Z"]

    def raw_split(yy, fix=True, swap=False):
        b = (yy - vmin) / dz
        lo, up = b.floor(), b.ceil()
        if fix:
            lo = torch.where((up > 0) & (lo == up), lo - 1, lo)
            up = torch.where((lo < Z - 1) & (lo == up), up + 1, up)
        ml, mu = (b - lo, up - b) if swap else (up - b, b - lo)
        out = torch.zeros(b.shape[0], Z + 2, dtype=torch.float64)
        out.scatter_add_(1, lo.long().clamp(0, Z + 1).unsqueeze(1), ml.unsqueeze(1))
        out.scatter_add_(1, up.long().clamp(0, Z + 1).unsqueeze(1), mu.unsqueeze(1))
        return out[:, :Z]
    r = C._d(inp["returns"])
    yb, _ = T.ybar(inp, astar)
    x = r + T.H.sc_of(inp) * yb
    slips = [("fix-ups dropped", raw_split(y, fix=False)), ("m_l and m_u swapped", raw_split(y, swap=True)),
             ("no clamp", raw_split((V.h(x, eps) if eps is not None else x).clamp(vmin - 5 * dz, vmax + 5 * dz)))]
    if eps is not None:
        slips.append(("h not applied", raw_split(x.clamp(vmin, vmax))))
    for name, got in slips:
        assert ((got - m).abs() / em).max() > 10, name
