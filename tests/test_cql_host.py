"""CQL(H)'s regulariser without a GPU: cql_options (args.cql_alpha) with its defaults and refusals, the two C entries'
signatures against the header and their host-side refusals, and tests/cql_ref.py -- its gradient against float64
autograd of the objective through the dueling combination, its limits (A = 1, R >= 0, the quantile head's zero
value-stream gradient) and its derived bound against an fp32 emulation of the kernels' operation order."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

import cql_ref as CQ
from test_qr_host import make_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RB_ERR_INVAL, RB_ERR_RANGE = -22, -34
ONE = 8   # a pointer that is never dereferenced: validation fails first
ENTRIES = ("rb_cql_grad", "rb_cql_dueling_grad")


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


# ---- options ---------------------------------------------------------------------------------------------------------------
def test_defaults_and_off():
    from rainbow_b200.agent import cql_options
    for off in (dict(), dict(cql_alpha=None), dict(cql_alpha=0), dict(cql_alpha=0.0)):
        assert cql_options(make_args(**off)) is None
    assert cql_options(make_args(cql_alpha=1)) == 1.0
    assert cql_options(make_args(cql_alpha=0.1)) == float(np.float32(0.1)), "rounded to the fp32 the kernels take"
    assert cql_options(make_args(cql_alpha=5.0, value_transform="none")) == 5.0


@pytest.mark.parametrize("bad", [-1.0, math.nan, math.inf, -math.inf, 1e-45, 1e39, "1", True])
def test_bad_alpha_is_refused(bad):
    from rainbow_b200.agent import cql_options
    with pytest.raises(ValueError, match="cql_alpha"):
        cql_options(make_args(cql_alpha=bad))


def test_value_rescaling_is_refused_naming_the_switch():
    from rainbow_b200.agent import cql_options
    with pytest.raises(ValueError, match="cql_alpha does not compose with value_transform 'rescale'"):
        cql_options(make_args(cql_alpha=1.0, value_transform="rescale"))


@pytest.mark.parametrize("extra", [dict(distribution="quantile"), dict(distribution="quantile", munchausen=True),
                                   dict(categorical_target="hl_gauss"), dict(categorical_target="two_hot"),
                                   dict(risk_measure="cvar"), dict(augment_m=2, augment_k=2),
                                   dict(augment_shift=4, target_tau=0.005, reset_interval=10, redo_interval=5,
                                        weight_decay=0.1, reset_optimizer=True, learn_stats=8, anneal_steps=100,
                                        bootstrap_truncation=True)])
def test_everything_else_composes(extra):
    from rainbow_b200.agent import cql_options
    assert cql_options(make_args(cql_alpha=2.0, **extra)) == 2.0


# ---- the C entries -----------------------------------------------------------------------------------------------------------
_CT = {"const float*": ctypes.c_void_p, "float*": ctypes.c_void_p, "const int64_t*": ctypes.c_void_p,
       "int": ctypes.c_int32, "float": ctypes.c_float, "rb_stream_t": ctypes.c_void_p}


def _header_decl(name):
    text = open(os.path.join(ROOT, "include", "rainbow_b200.h")).read()
    return re.search(r"int\s+" + name + r"\s*\(([^)]*)\)", text).group(1).split(",")


def _header_args(name):
    return [_CT[re.sub(r"\s*\w+$", "", a.strip()).replace(" *", "*")] for a in _header_decl(name)]


def _header_names(name):
    return [re.search(r"(\w+)$", a.strip()).group(1) for a in _header_decl(name)]


@pytest.mark.parametrize("name", ENTRIES)
def test_signatures_match_the_header(name):
    from rainbow_b200 import _lib
    ret, args = _lib.SIGNATURES[name]
    assert ret is ctypes.c_int and list(args) == _header_args(name)
    assert _header_names(name)[1:] == ["actions", "weights", "support", "alpha", "M", "B", "A", "Z",
                                       "dz" if "dueling" in name else "grad", "gap_out", "stream"]
    assert hasattr(lib(), name)
    assert lib().rb_abi_version() == 3, "additive entries: the ABI version stays"


def _good(name):
    names = _header_names(name)
    a = dict(zip(names, [ONE] * len(names)))
    a.update(alpha=1.0, M=1, B=4, A=6, Z=51, stream=None)
    return a, names


def _call(name, **over):
    a, names = _good(name)
    a.update(over)
    return getattr(lib(), name)(*[a[n] for n in names])


@pytest.mark.parametrize("name", ENTRIES)
def test_refusals_without_gpu(name):
    grad = "dz" if "dueling" in name else "grad"
    for ptr in (_header_names(name)[0], "actions", "weights", grad):
        assert _call(name, **{ptr: None}) == RB_ERR_INVAL, ptr
        msg = lib().rb_last_error().decode()
        assert msg.startswith(name) and "null" in msg, msg
    for field, bad in (("B", 0), ("B", -1), ("A", 0), ("A", -3), ("Z", 1), ("Z", 0)):
        assert _call(name, **{field: bad}) == RB_ERR_INVAL, (field, bad)
    for bad in (0.0, -1.0, math.nan, math.inf, -math.inf, 1e-40):   # 1e-40: subnormal
        assert _call(name, alpha=bad) == RB_ERR_INVAL, bad
        assert "alpha" in lib().rb_last_error().decode()
    assert _call(name, Z=129) == RB_ERR_RANGE
    for M in (0, -1, 9):
        assert _call(name, M=M) == RB_ERR_RANGE, M
    assert _call(name, A=4096, Z=128) == RB_ERR_RANGE, "rows too large for shared memory"
    assert "shared" in lib().rb_last_error().decode() or "large" in lib().rb_last_error().decode()
    assert _call(name, support=None, Z=129) == RB_ERR_RANGE, "the quantile head refuses the same shapes"


# ---- the reference -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("head", ["categorical", "quantile"])
@pytest.mark.parametrize("entry", ["plain", "dueling"])
@pytest.mark.parametrize("A,Z,M", [(6, 51, 1), (18, 5, 2), (3, 128, 4), (1, 51, 2)])
def test_gradient_is_autograd_of_the_objective(head, entry, A, Z, M):
    inp = CQ.make_inputs(entry, 7, A, Z, M, head, seed=A * 100 + Z + M)
    sup = None if inp["support"] is None else inp["support"].double()
    rows = inp["rows"].double().requires_grad_()
    if entry == "dueling":
        v, adv = rows[:, :Z].unsqueeze(1), rows[:, Z:].view(-1, A, Z)
        q = v + adv - adv.mean(1, keepdim=True)
    else:
        q = rows
    obj, _ = CQ.objective(q, inp["actions"], inp["weights"], sup, inp["alpha"], M)
    (want,) = torch.autograd.grad(obj, rows)
    out, _, _, _ = CQ.reference(inp)
    assert torch.allclose(out, want, rtol=1e-10, atol=1e-14)


@pytest.mark.parametrize("head", ["categorical", "quantile"])
@pytest.mark.parametrize("entry", ["plain", "dueling"])
def test_limits(head, entry):
    one = CQ.make_inputs(entry, 9, 1, 51, 2, head, seed=4)
    out, _, gap, _ = CQ.reference(one)
    assert torch.equal(gap, torch.zeros_like(gap)) and torch.equal(out, torch.zeros_like(out)), "A = 1: R = 0, no gradient"
    inp = CQ.make_inputs(entry, 33, 18, 51, 2, head, seed=5)
    out, _, gap, _ = CQ.reference(inp)
    assert bool((gap >= 0).all()), "logsumexp >= every Q_a"
    if head == "quantile":
        g, _, _, _, _ = CQ.grad_logits(CQ.logits(inp)[0], inp["actions"], inp["weights"], None, inp["alpha"], 2)
        assert float(g.sum(1).abs().max()) < 1e-18, "the value-stream gradient sum_a c (sigma_a - d_a) / N is 0"


@pytest.mark.parametrize("head", ["categorical", "quantile"])
@pytest.mark.parametrize("entry", ["plain", "dueling"])
@pytest.mark.parametrize("B,A,Z,M", [(5, 6, 51, 1), (3, 18, 101, 2), (4, 6, 2, 4), (2, 18, 128, 1), (6, 1, 64, 2)])
def test_fp32_emulation_is_within_the_bound(head, entry, B, A, Z, M):
    inp = CQ.make_inputs(entry, B, A, Z, M, head, seed=B * 1000 + Z + A + M, alpha=3.0)
    dz0 = torch.randn(inp["rows"].shape, generator=torch.Generator().manual_seed(Z)) * 1e-3
    out, e_out, gap, e_gap = CQ.reference(inp, dz0.float())
    em, eg = CQ.emulate(inp, dz0.float())
    d = (torch.from_numpy(em.astype(np.float64)).view_as(out) - out).abs()
    assert bool((d <= e_out).all()), float((d / e_out).max())
    dg = (torch.from_numpy(eg.astype(np.float64)) - gap).abs()
    assert bool((dg <= e_gap).all()), float((dg / e_gap).max())


def test_bound_sees_the_slips():
    """The slips DESIGN §22 lists move the output far past the bound: no max shift in sigma (overflow), the delta on the
    wrong action, = for +=, 1/B for 1/(M B), the value-stream sum dropped."""
    inp = CQ.make_inputs("dueling", 6, 6, 51, 2, "categorical", seed=9)
    dz0 = torch.randn(inp["rows"].shape, generator=torch.Generator().manual_seed(1)) * 1e-2
    out, e_out, _, _ = CQ.reference(inp, dz0)
    q = CQ.logits(inp)[0]
    sup = inp["support"].double()
    acts = inp["actions"]
    wrong = (acts + 1) % inp["A"]
    g_wrong, _, _, _, _ = CQ.grad_logits(q, wrong, inp["weights"], sup, inp["alpha"], 2)
    g_ok, _, _, _, _ = CQ.grad_logits(q, acts, inp["weights"], sup, inp["alpha"], 2)
    slips = {"delta on the wrong action": CQ.dueling_map(g_wrong) + dz0.double(),
             "= for +=": CQ.dueling_map(g_ok),
             "1/B for 1/(MB)": CQ.dueling_map(2 * g_ok) + dz0.double(),
             "value sum dropped": torch.cat([torch.zeros_like(g_ok.sum(1)),
                                             CQ.dueling_map(g_ok)[:, inp["Z"]:]], 1) + dz0.double()}
    for name, got in slips.items():
        assert ((got - out).abs() / e_out).max() > 10, name
