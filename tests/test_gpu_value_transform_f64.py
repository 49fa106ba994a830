"""Every value-rescaled entry point against the float64 reference of tests/vt_ref.py, per element: rb_qr_vt_loss_grad and
rb_qr_dueling_vt_loss_grad on vt_ref.QR_CASES, rb_c51_vt_loss_grad, rb_c51_dueling_vt_loss_grad and
rb_c51_dueling_avg_vt_loss_grad (K / M in {(1, 2), (2, 1), (2, 4)}) on C51_CASES, each at eps 0, 1e-3 and 1e-2, with
returns spanning |r| from 0 to 1e3, terminal rows, rows whose fp32 target lands exactly on an interior atom, ties and
weights 0 / 1; rb_qr_vt_q_values and
rb_learn_stats_batch_qr_vt.  Each loss case also checks graph replay = eager launch and NULL optional outputs bitwise.
h^-1 over ~2^20 fp32 values (+-0, subnormals, every binade to 1e6) runs through rb_qr_vt_q_values at N = 2, A = 1 (q =
h^-1(z_v) exactly: the dueling combination with zero advantages and the mean of two equal values are exact) and h over
the same values through theta_out of terminal rows (s = 0: T = h(r)), both within vt_ref.TAU_H relative."""
import numpy as np
import pytest
import torch

import c51_ref as C
import head_ref as R
import qr_ref as Q
import vt_ref as V
from test_gpu_head_f64 import graph_kernels
from test_gpu_parity import DEV

pytestmark = pytest.mark.gpu

NAN = float("nan")
GUARD = 3
EPS = [float(np.float32(e)) for e in V.EPS_GRID]


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


def stream():
    return torch.cuda.current_stream().cuda_stream


def ptr(t):
    return None if t is None else t.data_ptr()


def full(shape, v=NAN, dtype=torch.float32):
    return torch.full(shape, v, dtype=dtype, device=DEV)


# ---- QR ------------------------------------------------------------------------------------------------------------------
def run_qr(inp, with_outs=True):
    B, A, N, eps = inp["B"], inp["A"], inp["Z"], inp["eps"]
    ncol = A * N if inp["entry"] == "plain" else N + A * N
    loss, grad = full((B + GUARD,)), full((B + GUARD, ncol))
    T = full((B + GUARD, N)) if with_outs else None
    astar = full((B + GUARD,), -1, torch.int64) if with_outs else None
    common = (ptr(inp["actions"]), ptr(inp["returns"]), ptr(inp["nonterminals"]), ptr(inp["weights"]), C.f32(inp["kappa"]),
              C.f32(inp["gamma_n"]))
    L = lib()
    if inp["entry"] == "plain":
        rc = L.rb_qr_vt_loss_grad(ptr(inp["q_on_s"]), ptr(inp["q_on_ns"]), ptr(inp["q_tg_ns"]), *common, B, A, N,
                                  ptr(loss), ptr(grad), ptr(T), ptr(astar), eps, stream())
    else:
        rc = L.rb_qr_dueling_vt_loss_grad(ptr(inp["z_on"]), ptr(inp["z_tg"]), A, N, *common, B, ptr(loss), ptr(grad),
                                          ptr(T), ptr(astar), eps, stream())
    assert rc == 0, L.rb_last_error()
    return loss, grad, T, astar


QR = [(e, eps) + c for e in ("plain", "dueling") for c in V.QR_CASES for eps in EPS]


@pytest.mark.parametrize("case", QR, ids=[f"{e}-e{eps:g}-B{B}-A{A}-N{N}-k{k:g}" for e, eps, B, A, N, k in QR])
def test_qr_vt_f64(case, tmp_path):
    entry, eps, B, A, N, kappa = case
    inp = C.to(V.make_qr_inputs(entry, B, A, N, kappa, eps, seed=B * 1000 + A * 10 + N), DEV)
    eager = run_qr(inp)
    graph, outs, dot = graph_kernels(lambda: run_qr(inp), tmp_path / "qr.dot")
    assert ("k_qr_dueling" if entry == "dueling" else "k_qr") in dot
    for name, a, b in zip(("loss", "grad", "T", "astar"), eager, outs):
        assert torch.equal(a[:B], b[:B]), f"{name}: eager launch and graph replay differ"
        tail = b[B:]
        assert bool((tail == -1).all()) if b.dtype == torch.int64 else bool(torch.isnan(tail).all()), name
    bare = run_qr(inp, with_outs=False)
    assert torch.equal(bare[0][:B], outs[0][:B]) and torch.equal(bare[1][:B], outs[1][:B])
    loss, grad, T, astar = (t[:B] for t in outs)
    ev, evs = V.qr_mean_quantiles(inp)
    assert bool(Q.astar_ok(ev, evs, astar).all()), "a* is not within rounding of the best mean of h^-1"
    assert bool(C.first_of_identical(inp, astar).all())
    R.assert_within("T", T, *V.qr_targets(inp, astar), Q.TAU)
    (l_ref, l_scale), (g_ref, g_scale) = Q.loss_grad(inp, T)
    R.assert_within("loss", loss, l_ref, l_scale, Q.TAU)
    assert bool((grad[inp["weights"] == 0] == 0).all())
    if entry == "plain":
        g3 = grad.view(B, A, N)
        R.assert_within("grad", g3[torch.arange(B, device=DEV), inp["actions"]], g_ref, g_scale, Q.TAU)
    else:
        R.assert_within("dz", grad, *C.dueling_dz(inp, g_ref, g_scale), Q.TAU)


@pytest.mark.parametrize("eps", EPS)
@pytest.mark.parametrize("M,A,N", [(1, 6, 51), (37, 18, 128), (5, 1, 2), (130, 64, 33)])
def test_qr_vt_q_values_f64(M, A, N, eps):
    g = torch.Generator().manual_seed(M * 100 + A + N)
    z = torch.randn(M, N + A * N, generator=g) * 5.0
    tied = torch.arange(M) % 3 == 1
    z[tied, N:] = z[tied, N:2 * N].repeat(1, A)
    z = z.to(DEV)
    q, best_a, best_q = full((M + GUARD, A)), full((M + GUARD,), -1, torch.int64), full((M + GUARD,))
    L = lib()
    assert L.rb_qr_vt_q_values(ptr(z), M, A, N, ptr(q), ptr(best_a), ptr(best_q), eps, stream()) == 0
    torch.cuda.synchronize()
    assert bool(torch.isnan(q[M:]).all()) and bool((best_a[M:] == -1).all())
    q, best_a, best_q = q[:M], best_a[:M], best_q[:M]
    ev, scale = V.qr_q_values(z, A, N, eps)
    R.assert_within("q", q, ev, scale, Q.TAU_EV)
    assert bool((best_a[tied.to(DEV)] == 0).all())
    assert torch.equal(best_q, q[torch.arange(M, device=DEV), best_a]) and torch.equal(q.argmax(1), best_a)


def _sweep_values():
    """~2^20 fp32 values: +-0, subnormals and every binade up to 1e6, evenly spaced in the bit patterns."""
    top = int(np.array(1e6, dtype=np.float32).view(np.int32))
    bits = np.unique(np.concatenate([np.arange(0, top, top // (1 << 19), dtype=np.int64), [0, 1, 2, 0x7FFFFF, 0x800000,
                                                                                          top]]))
    pos = bits.astype(np.int32).view(np.float32)
    return torch.from_numpy(np.concatenate([pos, -pos]))


@pytest.mark.parametrize("eps", EPS + [1.0])
def test_hinv_and_h_elementwise(eps):
    v = _sweep_values()
    M = v.numel()
    L = lib()
    z = torch.zeros(M, 2 + 2)
    z[:, 0] = z[:, 1] = v                   # z_v = (v, v), z_a = 0 at A = 1
    z = z.to(DEV)
    q = full((M, 1))
    assert L.rb_qr_vt_q_values(ptr(z), M, 1, 2, ptr(q), None, None, eps, stream()) == 0
    ref = V.hinv(v.double(), eps).to(DEV)
    err = (q[:, 0].double() - ref).abs()
    assert bool((err <= V.TAU_H * ref.abs() + V.SUB_FLOOR).all()), f"h^-1: worst {float((err / ref.abs()).nan_to_num().max())}"
    # h through theta_out of terminal rows: T = h(fl32(r + 0)) = h(r)
    B = M
    rows = torch.zeros(B, 1, 2, device=DEV)
    T = full((B, 2))
    loss, grad = full((B,)), full((B, 2))
    acts = torch.zeros(B, dtype=torch.int64, device=DEV)
    nts, w = torch.zeros(B, device=DEV), torch.ones(B, device=DEV)
    rets = v.to(DEV)
    assert L.rb_qr_vt_loss_grad(ptr(rows), ptr(rows), ptr(rows), ptr(acts), ptr(rets), ptr(nts), ptr(w), 1.0, 0.99, B, 1, 2,
                                ptr(loss), ptr(grad), ptr(T), None, eps, stream()) == 0
    ref = V.h(v.double(), eps).to(DEV)
    err = (T[:, 0].double() - ref).abs()
    assert bool((err <= V.TAU_H * ref.abs() + V.SUB_FLOOR).all()), f"h: worst {float((err / ref.abs()).nan_to_num().max())}"
    assert torch.equal(T[:, 0], T[:, 1])


@pytest.mark.parametrize("eps", EPS)
@pytest.mark.parametrize("layout", ["z", "q"])
def test_learn_stats_qr_vt(layout, eps):
    """q_mean and target_mean of the record in return units: mean_b mean_i h^-1 of the online quantiles of the taken
    action and of the kernel's T rows."""
    B, A, N = 70, 6, 51
    inp = C.to(V.make_qr_inputs("dueling" if layout == "z" else "plain", B, A, N, 1.0, eps, seed=7), DEV)
    loss, grad, T, astar = (t[:B] for t in run_qr(inp))
    scratch = torch.zeros(lib().rb_learn_stats_scratch_elems(), dtype=torch.float64, device=DEV)
    z = inp["z_on"] if layout == "z" else None
    q = inp["q_on_s"] if layout == "q" else None
    assert lib().rb_learn_stats_batch_qr_vt(ptr(loss), ptr(inp["weights"]), ptr(inp["actions"]), ptr(T), ptr(z), ptr(q), B,
                                            A, N, ptr(scratch), eps, stream()) == 0
    torch.cuda.synchronize()
    qs, _ = C.logits(inp, "s")
    theta = C._row(qs, inp["actions"])
    q_mean = float(V.hinv(theta, eps).mean())
    t_mean = float(V.hinv(T.double(), eps).mean())
    scale_q = float(V.hinv(theta, eps).abs().mean()) + 1e-30
    scale_t = float(V.hinv(T.double(), eps).abs().mean()) + 1e-30
    assert abs(float(scratch[2]) - q_mean) <= 1e-5 * scale_q
    assert abs(float(scratch[3]) - t_mean) <= 1e-5 * scale_t
    assert float(scratch[0]) == pytest.approx(float(loss.double().mean()), rel=1e-6)


# ---- C51 -----------------------------------------------------------------------------------------------------------------
C51_SHAPES = [(32, 6, 51), (5, 2, 2), (33, 6, 31), (35, 1, 32), (1, 64, 33), (512, 6, 51), (5, 6, 65), (3, 18, 128),
              (2048, 6, 51), (1, 1, 128), (35, 2, 128), (33, 18, 64)]


def run_c51(inp, with_outs=True, MK=None):
    B, A, Z, eps = inp["B"], inp["A"], inp["Z"], inp["eps"]
    entry = inp["entry"]
    M, K = MK or (1, 1)
    ncol = A * Z if entry == "plain" else Z + A * Z
    loss, grad = full((B + GUARD,)), full((M * B + GUARD, ncol))
    m = full((B + GUARD, Z)) if with_outs else None
    astar = full((K * B + GUARD,), -1, torch.int64) if with_outs else None
    sup = (ptr(inp["support"]), C.f32(inp["vmin"]), C.f32(inp["vmax"]), C.f32(inp["dz"]), C.f32(inp["gamma_n"]))
    rows = (ptr(inp["actions"]), ptr(inp["returns"]), ptr(inp["nonterminals"]), ptr(inp["weights"]))
    L = lib()
    if entry == "plain":
        rc = L.rb_c51_vt_loss_grad(ptr(inp["q_on_s"]), ptr(inp["q_on_ns"]), ptr(inp["q_tg_ns"]), *rows, *sup, B, A, Z,
                                   ptr(loss), ptr(grad), ptr(m), ptr(astar), ptr(inp["support_q"]), eps, stream())
    elif MK is None:
        rc = L.rb_c51_dueling_vt_loss_grad(ptr(inp["z_on"]), ptr(inp["z_tg"]), A, Z, *rows, *sup, B, ptr(loss), ptr(grad),
                                           ptr(m), ptr(astar), ptr(inp["support_q"]), eps, stream())
    else:
        rc = L.rb_c51_dueling_avg_vt_loss_grad(ptr(inp["z_on"]), ptr(inp["z_tg"]), A, Z, *rows, *sup, B, M, K, ptr(loss),
                                               ptr(grad), ptr(m), ptr(astar), ptr(inp["support_q"]), eps, stream())
    assert rc == 0, L.rb_last_error()
    return loss, grad, m, astar


C51 = [(e, eps) + c for e in ("plain", "dueling") for c in C51_SHAPES for eps in EPS]


@pytest.mark.parametrize("case", C51, ids=[f"{e}-e{eps:g}-B{B}-A{A}-Z{Z}" for e, eps, B, A, Z in C51])
def test_c51_vt_f64(case, tmp_path):
    entry, eps, B, A, Z = case
    inp = C.to(V.make_c51_inputs(entry, B, A, Z, eps, seed=B * 1000 + A * 10 + Z), DEV)
    eager = run_c51(inp)
    graph, outs, dot = graph_kernels(lambda: run_c51(inp), tmp_path / "c51.dot")
    assert ("k_c51_dueling" if entry == "dueling" else "k_c51") in dot
    n_on = sum(C.RET_KINDS[i % 5] == "on_atom" for i in range(B))
    if Z > 2:        # at Z = 2 both atoms are end atoms, which the below / above rows reach through the clamp
        assert inp["on_atom"] == n_on, "every on_atom row's target lands exactly on an interior atom"
    for name, a, b in zip(("loss", "grad", "m", "astar"), eager, outs):
        assert torch.equal(a[:B], b[:B]), f"{name}: eager launch and graph replay differ"
        tail = b[B:]
        assert bool((tail == -1).all()) if b.dtype == torch.int64 else bool(torch.isnan(tail).all()), \
            f"{name}: written past its last row"
    bare = run_c51(inp, with_outs=False)
    assert torch.equal(bare[0][:B], outs[0][:B]) and torch.equal(bare[1][:B], outs[1][:B])
    loss, grad, m, astar = (t[:B] for t in outs)
    ev, evs = V.c51_expected_values(inp)
    assert bool(C.astar_ok(ev, evs, astar).all()), "a* is not within rounding of the best expected return"
    assert bool(C.first_of_identical(inp, astar).all())
    R.assert_within("m", m, *V.c51_projection(inp, astar), C.TAU)
    (l_ref, l_scale), (g_ref, g_scale) = C.loss_grad(inp, m)
    R.assert_within("loss", loss, l_ref, l_scale, C.TAU)
    if entry == "plain":
        R.assert_within("grad", grad.view(B, A, Z)[torch.arange(B, device=DEV), inp["actions"]], g_ref, g_scale, C.TAU)
    else:
        R.assert_within("dz", grad, *C.dueling_dz(inp, g_ref, g_scale), C.TAU)


@pytest.mark.parametrize("eps", EPS)
@pytest.mark.parametrize("MK", [(1, 1), (1, 2), (2, 1), (2, 4)])
def test_c51_avg_vt_f64(MK, eps):
    """The averaging entry: at M = K = 1 bitwise the dueling entry; otherwise m = mean_k of the per-copy transformed
    projections (each at the kernel's a*_k) and loss = mean_j of the per-copy losses against the kernel's m."""
    M, K = MK
    B, A, Z = 35, 6, 51
    base = V.make_c51_inputs("dueling", B, A, Z, eps, seed=11)
    g = torch.Generator().manual_seed(12)
    ncol = Z + A * Z
    s_rows = [base["z_on"][:B]] + [torch.randn(B, ncol, generator=g) * 2 for _ in range(M - 1)]
    ns_rows = [base["z_on"][B:]] + [torch.randn(B, ncol, generator=g) * 2 for _ in range(K - 1)]
    t_rows = [base["z_tg"]] + [torch.randn(B, ncol, generator=g) * 2 for _ in range(K - 1)]
    inp = C.to(dict(base, z_on=torch.cat(s_rows + ns_rows), z_tg=torch.cat(t_rows)), DEV)
    loss, dz, m, astar = run_c51(inp, MK=MK)
    if MK == (1, 1):
        one = run_c51(C.to(base, DEV))
        for a, b in zip((loss, dz, m, astar), one):
            assert torch.equal(a[:B], b[:B])
        return
    loss, m = loss[:B], m[:B]
    mk, sk = [], []
    for k in range(K):
        ik = dict(inp, z_on=torch.cat([s_rows[0].to(DEV), ns_rows[k].to(DEV)]), z_tg=t_rows[k].to(DEV))
        ak = astar[k * B:(k + 1) * B]
        ev, evs = V.c51_expected_values(ik)
        assert bool(C.astar_ok(ev, evs, ak).all())
        a, b = V.c51_projection(ik, ak)
        mk.append(a)
        sk.append(b)
    R.assert_within("m", m, sum(mk) / K, sum(sk) / K + sum(x.abs() for x in mk) / K, C.TAU)
    ls, lss = 0.0, 0.0
    for j in range(M):
        ij = dict(inp, z_on=torch.cat([s_rows[j].to(DEV), ns_rows[0].to(DEV)]), z_tg=t_rows[0].to(DEV))
        (lj, sj), _ = C.loss_grad(ij, m)
        ls, lss = ls + lj, lss + sj + lj.abs()
    R.assert_within("loss", loss, ls / M, lss / M, C.TAU)
