"""The distributional loss through both C entry points (rb_c51_loss_grad -> k_c51<R>, rb_c51_dueling_loss_grad ->
k_c51_dueling<R>, R = 2 up to 64 atoms, 4 up to 128) against the float64 reference of tests/c51_ref.py, per element
(|err| <= TAU * scale; the arg-max within TAU_EV of the best expected value), on the grid c51_ref.CASES: atoms 2 to 128
across the R switch, actions 1 to 64, batches 1 to 2048, five supports (two where b rounds past Z - 1 at Vmax) and the
decreasing one (the projection's full-scan branch), with every row kind of c51_ref.make_inputs in the larger batches
(terminal rows, returns clamped to Vmin and to Vmax, returns on an atom, weights 0 and 1, sharp / constant / tied logits).
Each case captures its call as a CUDA graph and asserts from the graph's kernel nodes which variant ran, prefills the
outputs with NaN (a* with -1) and keeps guard rows past the batch that must stay untouched, requires a* of tied rows to be
the first action exactly and the gradient rows of the actions not taken (plain entry point) to be exactly 0, and requires
an eager launch, the graph replay and a launch without m_out / astar_out to agree bitwise.  Observed largest |err| / scale
per output and variant go to $RB_PARITY_OBSERVED when that variable is set."""
import re

import pytest
import torch

import c51_ref as C
import head_ref as R
from test_gpu_head_f64 import graph_kernels, record
from test_gpu_parity import DEV

pytestmark = pytest.mark.gpu

NAN = float("nan")
GUARD = 3
RB_ERR_RANGE = -34


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


def stream():
    return torch.cuda.current_stream().cuda_stream


_K = re.compile(r"k_c51(_dueling)?(?:<\s*(\d)\s*>|ILi(\d)E)")


def variants_of(dot):
    return {f"k_c51{d}<{a or b}>" for d, a, b in _K.findall(dot)}


def run(inp, with_m=True):
    """One launch into NaN-prefilled outputs with GUARD rows; returns (loss, grad or dz, m, astar) with the guard rows."""
    B, A, Z = inp["B"], inp["A"], inp["Z"]
    ncol = A * Z if inp["entry"] == "plain" else Z + A * Z
    loss = torch.full((B + GUARD,), NAN, device=DEV)
    grad = torch.full((B + GUARD, ncol), NAN, device=DEV)
    m = torch.full((B + GUARD, Z), NAN, device=DEV) if with_m else None
    astar = torch.full((B + GUARD,), -1, dtype=torch.int64, device=DEV) if with_m else None
    ptr = lambda t: None if t is None else t.data_ptr()
    tail = (C.f32(inp["vmin"]), C.f32(inp["vmax"]), C.f32(inp["dz"]), C.f32(inp["gamma_n"]))
    common = (inp["actions"].data_ptr(), inp["returns"].data_ptr(), inp["nonterminals"].data_ptr(), inp["weights"].data_ptr(),
              inp["support"].data_ptr()) + tail
    L = lib()
    if inp["entry"] == "plain":
        rc = L.rb_c51_loss_grad(inp["q_on_s"].data_ptr(), inp["q_on_ns"].data_ptr(), inp["q_tg_ns"].data_ptr(), *common, B, A, Z,
                                loss.data_ptr(), grad.data_ptr(), ptr(m), ptr(astar), stream())
    else:
        rc = L.rb_c51_dueling_loss_grad(inp["z_on"].data_ptr(), inp["z_tg"].data_ptr(), A, Z, *common, B, loss.data_ptr(),
                                        grad.data_ptr(), ptr(m), ptr(astar), stream())
    assert rc == 0, L.rb_last_error()
    return loss, grad, m, astar


def _guard_untouched(name, t, B):
    tail = t[B:]
    ok = bool((tail == -1).all()) if t.dtype == torch.int64 else bool(torch.isnan(tail).all())
    assert ok, f"{name}: written past its last row"


CASES = [(e,) + c for e in ("plain", "dueling") for c in C.CASES]


@pytest.mark.parametrize("case", CASES, ids=[f"{e}-B{B}-A{A}-Z{Z}-{s}" for e, B, A, Z, s in CASES])
def test_c51_f64(case, tmp_path):
    entry, B, A, Z, sup = case
    inp = C.to(C.make_inputs(entry, B, A, Z, sup, seed=B * 1000 + A * 10 + Z), DEV)
    eager = run(inp)
    graph, outs, dot = graph_kernels(lambda: run(inp), tmp_path / "c51.dot")
    variant = ("k_c51_dueling" if entry == "dueling" else "k_c51") + ("<2>" if Z <= 64 else "<4>")
    assert variants_of(dot) == {variant}, f"kernels launched {variants_of(dot)}, expected {variant}"
    loss, grad, m, astar = outs
    for name, t in zip(("loss", "grad", "m", "astar"), outs):
        _guard_untouched(name, t, B)
    for name, a, b in zip(("loss", "grad", "m", "astar"), eager, outs):
        assert torch.equal(a[:B], b[:B]), f"{name}: eager launch and graph replay differ"
    bare = run(inp, with_m=False)
    assert torch.equal(bare[0][:B], loss[:B]) and torch.equal(bare[1][:B], grad[:B]), "m_out / astar_out NULL changes the result"
    loss, grad, m, astar = loss[:B], grad[:B], m[:B], astar[:B]

    assert bool(((astar >= 0) & (astar < A)).all()), "a* in range"
    ev, evs = C.expected_values(inp)
    assert bool(C.astar_ok(ev, evs, astar).all()), "a* is not within rounding of the best expected value"
    assert bool(C.first_of_identical(inp, astar).all()), "a tie of identical rows goes to the first action"
    m_ref, m_scale = C.projection(inp, astar)
    record(f"c51.{variant}.m", R.assert_within("m", m, m_ref, m_scale, C.TAU))
    (l_ref, l_scale), (g_ref, g_scale) = C.loss_grad(inp, m)
    record(f"c51.{variant}.loss", R.assert_within("loss", loss, l_ref, l_scale, C.TAU))
    acts = inp["actions"]
    if entry == "plain":
        g3 = grad.view(B, A, Z)
        taken = torch.zeros(B, A, dtype=torch.bool, device=DEV)
        taken[torch.arange(B, device=DEV), acts] = True
        assert bool((g3[~taken] == 0).all()), "gradient rows of the actions not taken are exactly 0"
        record(f"c51.{variant}.grad", R.assert_within("grad", g3[taken], g_ref, g_scale, C.TAU))
    else:
        dz_ref, dz_scale = C.dueling_dz(inp, g_ref, g_scale)
        record(f"c51.{variant}.dz", R.assert_within("dz", grad, dz_ref, dz_scale, C.TAU))


@pytest.mark.parametrize("A,rc", [(130, 0), (131, RB_ERR_RANGE)])
def test_c51_dueling_shared_memory_limit(A, rc):
    """At 128 atoms the dueling kernel's dynamic shared memory, (3 (Z + A Z) + 3 Z + A) floats, is 203 272 B at 130
    actions (accepted, and checked against the reference) and 204 812 B at 131 (over 200 KB: RB_ERR_RANGE, nothing
    written)."""
    B, Z = 3, 128
    assert (3 * (Z + A * Z) + 3 * Z + A) * 4 == {130: 203272, 131: 204812}[A]
    inp = C.to(C.make_inputs("dueling", B, A, Z, "pm10", seed=A), DEV)
    if rc == 0:
        loss, dz, m, astar = (t[:B] for t in run(inp))
        ev, evs = C.expected_values(inp)
        assert bool(C.astar_ok(ev, evs, astar).all()) and bool(C.first_of_identical(inp, astar).all())
        m_ref, m_scale = C.projection(inp, astar)
        R.assert_within("m", m, m_ref, m_scale, C.TAU)
        (l_ref, l_scale), (g_ref, g_scale) = C.loss_grad(inp, m)
        R.assert_within("loss", loss, l_ref, l_scale, C.TAU)
        R.assert_within("dz", dz, *C.dueling_dz(inp, g_ref, g_scale), C.TAU)
        return
    ncol = Z + A * Z
    loss = torch.full((B,), NAN, device=DEV)
    dz = torch.full((B, ncol), NAN, device=DEV)
    m = torch.full((B, Z), NAN, device=DEV)
    astar = torch.full((B,), -1, dtype=torch.int64, device=DEV)
    L = lib()
    got = L.rb_c51_dueling_loss_grad(inp["z_on"].data_ptr(), inp["z_tg"].data_ptr(), A, Z, inp["actions"].data_ptr(),
                                     inp["returns"].data_ptr(), inp["nonterminals"].data_ptr(), inp["weights"].data_ptr(),
                                     inp["support"].data_ptr(), -10.0, 10.0, C.f32(inp["dz"]), C.f32(inp["gamma_n"]), B,
                                     loss.data_ptr(), dz.data_ptr(), m.data_ptr(), astar.data_ptr(), stream())
    torch.cuda.synchronize()
    assert got == rc, L.rb_last_error()
    assert all(bool(torch.isnan(t).all()) for t in (loss, dz, m)) and bool((astar == -1).all()), "a refused call writes nothing"

