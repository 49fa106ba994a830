"""The quantile-regression loss through both C entry points (rb_qr_loss_grad -> k_qr<R>, rb_qr_dueling_loss_grad ->
k_qr_dueling<R>, R = 2 up to 64 quantiles, 4 up to 128) and rb_qr_q_values against the float64 reference of
tests/qr_ref.py, per element (|err| <= TAU * scale; a* within TAU_EV of the best mean), on the grid qr_ref.CASES: N 2 to
128 across the R switch, A 1 to 64, B 1 to 2048, kappa 0.25 / 1 / 10, with every row kind of qr_ref.make_inputs (terminal
rows, all |u| < kappa, all |u| > kappa, constant rows, ties, weights 0 and 1).  Each case captures its call as a CUDA
graph and reads the variant that ran from the graph's kernel nodes, prefills the outputs with NaN (a* with -1) and keeps
guard rows past the batch that must stay untouched, requires a* of tied rows to be the first action exactly, the rows of
weight 0 and (plain entry point) the rows of the actions not taken to be exactly 0, and an eager launch, the graph replay
and a launch without theta_out / astar_out to agree bitwise."""
import re

import pytest
import torch

import c51_ref as C
import head_ref as R
import qr_ref as Q
from test_gpu_head_f64 import graph_kernels
from test_gpu_parity import DEV

pytestmark = pytest.mark.gpu

NAN = float("nan")
GUARD = 3


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


def stream():
    return torch.cuda.current_stream().cuda_stream


_K = re.compile(r"k_qr(_dueling)?(?:<\s*(\d)\s*>|ILi(\d)E)")


def variants_of(dot):
    return {f"k_qr{d}<{a or b}>" for d, a, b in _K.findall(dot)}


def run(inp, with_outs=True):
    """One launch into NaN-prefilled outputs with GUARD rows; returns (loss, grad or dz, T, astar) with the guard rows."""
    B, A, N = inp["B"], inp["A"], inp["Z"]
    ncol = A * N if inp["entry"] == "plain" else N + A * N
    loss = torch.full((B + GUARD,), NAN, device=DEV)
    grad = torch.full((B + GUARD, ncol), NAN, device=DEV)
    T = torch.full((B + GUARD, N), NAN, device=DEV) if with_outs else None
    astar = torch.full((B + GUARD,), -1, dtype=torch.int64, device=DEV) if with_outs else None
    ptr = lambda t: None if t is None else t.data_ptr()
    common = (inp["actions"].data_ptr(), inp["returns"].data_ptr(), inp["nonterminals"].data_ptr(), inp["weights"].data_ptr(),
              C.f32(inp["kappa"]), C.f32(inp["gamma_n"]))
    L = lib()
    if inp["entry"] == "plain":
        rc = L.rb_qr_loss_grad(inp["q_on_s"].data_ptr(), inp["q_on_ns"].data_ptr(), inp["q_tg_ns"].data_ptr(), *common, B, A, N,
                               loss.data_ptr(), grad.data_ptr(), ptr(T), ptr(astar), stream())
    else:
        rc = L.rb_qr_dueling_loss_grad(inp["z_on"].data_ptr(), inp["z_tg"].data_ptr(), A, N, *common, B, loss.data_ptr(),
                                       grad.data_ptr(), ptr(T), ptr(astar), stream())
    assert rc == 0, L.rb_last_error()
    return loss, grad, T, astar


def _guard_untouched(name, t, B):
    tail = t[B:]
    ok = bool((tail == -1).all()) if t.dtype == torch.int64 else bool(torch.isnan(tail).all())
    assert ok, f"{name}: written past its last row"


CASES = [(e,) + c for e in ("plain", "dueling") for c in Q.CASES]


@pytest.mark.parametrize("case", CASES, ids=[f"{e}-B{B}-A{A}-N{N}-k{k:g}" for e, B, A, N, k in CASES])
def test_qr_f64(case, tmp_path):
    entry, B, A, N, kappa = case
    inp = C.to(Q.make_inputs(entry, B, A, N, kappa, seed=B * 1000 + A * 10 + N), DEV)
    eager = run(inp)
    graph, outs, dot = graph_kernels(lambda: run(inp), tmp_path / "qr.dot")
    variant = ("k_qr_dueling" if entry == "dueling" else "k_qr") + ("<2>" if N <= 64 else "<4>")
    assert variants_of(dot) == {variant}, f"kernels launched {variants_of(dot)}, expected {variant}"
    for name, t in zip(("loss", "grad", "T", "astar"), outs):
        _guard_untouched(name, t, B)
    for name, a, b in zip(("loss", "grad", "T", "astar"), eager, outs):
        assert torch.equal(a[:B], b[:B]), f"{name}: eager launch and graph replay differ"
    bare = run(inp, with_outs=False)
    assert torch.equal(bare[0][:B], outs[0][:B]) and torch.equal(bare[1][:B], outs[1][:B]), \
        "theta_out / astar_out NULL changes the result"
    loss, grad, T, astar = (t[:B] for t in outs)

    assert bool(((astar >= 0) & (astar < A)).all()), "a* in range"
    ev, evs = Q.mean_quantiles(inp)
    assert bool(Q.astar_ok(ev, evs, astar).all()), "a* is not within rounding of the best mean quantile"
    assert bool(C.first_of_identical(inp, astar).all()), "a tie of identical rows goes to the first action"
    R.assert_within("T", T, *Q.targets(inp, astar), Q.TAU)
    (l_ref, l_scale), (g_ref, g_scale) = Q.loss_grad(inp, T)
    R.assert_within("loss", loss, l_ref, l_scale, Q.TAU)
    assert bool((loss >= 0).all())
    zero_w = inp["weights"] == 0
    assert bool((grad[zero_w] == 0).all()), "rows of weight 0 have an exactly zero gradient"
    acts = inp["actions"]
    if entry == "plain":
        g3 = grad.view(B, A, N)
        taken = torch.zeros(B, A, dtype=torch.bool, device=DEV)
        taken[torch.arange(B, device=DEV), acts] = True
        assert bool((g3[~taken] == 0).all()), "gradient rows of the actions not taken are exactly 0"
        R.assert_within("grad", g3[taken], g_ref, g_scale, Q.TAU)
    else:
        R.assert_within("dz", grad, *C.dueling_dz(inp, g_ref, g_scale), Q.TAU)


@pytest.mark.parametrize("M,A,N", [(1, 6, 51), (37, 18, 128), (5, 1, 2), (130, 64, 33)])
def test_qr_q_values_f64(M, A, N):
    """rb_qr_q_values: q within TAU_EV of the float64 mean quantile, the arg-max within rounding of the best and the first
    of identical rows exactly, best_q = q[best_action] bitwise; the three outputs are each optional."""
    g = torch.Generator().manual_seed(M * 100 + A + N)
    z = torch.randn(M, N + A * N, generator=g) * 2.0
    tied = torch.arange(M) % 3 == 1                      # every advantage row equal: all actions tie
    z[tied, N:] = z[tied, N:2 * N].repeat(1, A)
    z = z.to(DEV)
    q = torch.full((M + GUARD, A), NAN, device=DEV)
    best_a = torch.full((M + GUARD,), -1, dtype=torch.int64, device=DEV)
    best_q = torch.full((M + GUARD,), NAN, device=DEV)
    L = lib()
    assert L.rb_qr_q_values(z.data_ptr(), M, A, N, q.data_ptr(), best_a.data_ptr(), best_q.data_ptr(), stream()) == 0
    torch.cuda.synchronize()
    assert bool(torch.isnan(q[M:]).all()) and bool((best_a[M:] == -1).all()) and bool(torch.isnan(best_q[M:]).all())
    q, best_a, best_q = q[:M], best_a[:M], best_q[:M]
    ev, scale = Q.q_values(z, A, N)
    R.assert_within("q", q, ev, scale, Q.TAU_EV)
    assert bool(Q.astar_ok(ev, scale, best_a).all())
    assert bool((best_a[tied.to(DEV)] == 0).all()), "ties go to the first action"
    assert torch.equal(best_q, q[torch.arange(M, device=DEV), best_a])
    assert torch.equal(q.argmax(1), best_a), "the first maximum of the kernel's own values"
    a_only = torch.full((M,), -1, dtype=torch.int64, device=DEV)
    assert L.rb_qr_q_values(z.data_ptr(), M, A, N, None, a_only.data_ptr(), None, stream()) == 0
    torch.cuda.synchronize()
    assert torch.equal(a_only, best_a)
