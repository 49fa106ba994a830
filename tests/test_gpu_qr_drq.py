"""DrQ's K / M averaging under the quantile loss on the GPU (rb_qr_dueling_avg_loss_grad -> k_qr_dueling_avg<R, false>,
rb_qr_dueling_avg_vt_loss_grad -> k_qr_dueling_avg<R, true>, args.quantile_average_copies).

* The kernel: a*_k, Tbar, the loss and every dz element against tests/qr_drq_ref.py (|err| <= qr_ref.TAU x scale, the
  scales widened by the k-sum, / K and / M roundings), over N 2 to 128 across the R switch at 64, A 1 / 6 / 18, B 1 to
  512, (M, K) from (1, 2) to (8, 8), kappa 0.25 / 1 / 10 and value rescaling at eps 0 and 1e-3, with qr_ref's row kinds
  (terminals, ties, weight 0).  Outputs are prefilled with NaN / -1 and guard rows past each must stay untouched; the
  template variant is read from a captured graph's nodes, and the graph replay, the eager launch and a launch without the
  optional outputs agree bitwise.  At M = K = 1 every output is rb_qr_dueling(_vt)_loss_grad's bitwise; K (or M)
  identical copies, K a power of two up to 4, give Tbar = T (loss = loss) bitwise.  An over-size call is refused and
  writes nothing.
* The learner: identical copies (pad 0, intensity 0, M = K = 2) give a plain quantile agent's loss, T and priorities
  bitwise and its gradient within 5e-7 of its largest element; graph replays equal eager updates; the update graph is the
  quantile graph with k_qr_dueling_avg in place of k_qr_dueling (and the large-batch head backward for M B rows); the
  switch at M = K = 1 leaves the graph as it is; resume equals never stopping and a mismatched switch is refused before
  anything is restored; the statistics hold the averaged loss and Tbar's mean; acting is unaugmented; the library head
  with copies is refused.  Under value rescaling, the learner's loss, Tbar and dz of one fused M = K = 2 update against the
  vt_ref-based reference on its own head rows.
* Whole updates: tests/test_gpu_update_f64.py's trajectory check, unchanged, over four more cases pairing quantile x DrQ
  with every level of horizon, optimiser, target, reset, ReDo, statistics, net, noise and batch 1 / 32 / 33 / 64.
Deterministic cuDNN, like the other trajectory tests."""
import json
import re

import numpy as np
import pytest
import torch

import c51_ref as C
import head_ref as R
import qr_drq_ref as QD
import qr_ref as Q
import test_gpu_update_f64 as TU
from helpers import assert_bits_equal
from test_gpu_augment import update_graph
from test_gpu_head_f64 import graph_kernels
from test_gpu_parity import DEV, FakeEnv, cpu, make_args, synthetic_ring
from update_cases import _row, case_id

pytestmark = pytest.mark.gpu

NAN = float("nan")
GUARD = 3
CAP = 8192


@pytest.fixture(autouse=True)
def deterministic_cudnn():
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = old


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


def stream():
    return torch.cuda.current_stream().cuda_stream


_K = re.compile(r"k_qr_dueling(_avg)?(?:<\s*(\d)\s*,|ILi(\d)E)")


def variants_of(dot):
    return {f"k_qr_dueling{d}<{a or b}>" for d, a, b in _K.findall(dot)}


def run_avg(inp, with_outs=True):
    """One launch into NaN-prefilled outputs with GUARD rows past each: (loss, dz, T, astar), guards included."""
    B, A, N, M, K = inp["B"], inp["A"], inp["Z"], inp["M"], inp["K"]
    loss = torch.full((B + GUARD,), NAN, device=DEV)
    dz = torch.full((M * B + GUARD, N + A * N), NAN, device=DEV)
    T = torch.full((B + GUARD, N), NAN, device=DEV) if with_outs else None
    astar = torch.full((K * B + GUARD,), -1, dtype=torch.int64, device=DEV) if with_outs else None
    ptr = lambda t: None if t is None else t.data_ptr()
    args = (inp["z_on"].data_ptr(), inp["z_tg"].data_ptr(), A, N, inp["actions"].data_ptr(), inp["returns"].data_ptr(),
            inp["nonterminals"].data_ptr(), inp["weights"].data_ptr(), C.f32(inp["kappa"]), C.f32(inp["gamma_n"]), B, M, K,
            loss.data_ptr(), dz.data_ptr(), ptr(T), ptr(astar))
    L = lib()
    if inp.get("eps") is None:
        rc = L.rb_qr_dueling_avg_loss_grad(*args, stream())
    else:
        rc = L.rb_qr_dueling_avg_vt_loss_grad(*args, inp["eps"], stream())
    assert rc == 0, L.rb_last_error()
    return loss, dz, T, astar


def run_single(inp):
    """rb_qr_dueling(_vt)_loss_grad on online copy 0 and target copy 0: (loss, dz, T, astar)."""
    B, A, N = inp["B"], inp["A"], inp["Z"]
    one = QD.single(inp)
    loss, dz = torch.empty(B, device=DEV), torch.empty((B, N + A * N), device=DEV)
    T, astar = torch.empty((B, N), device=DEV), torch.empty(B, dtype=torch.int64, device=DEV)
    args = (one["z_on"].data_ptr(), one["z_tg"].data_ptr(), A, N, inp["actions"].data_ptr(), inp["returns"].data_ptr(),
            inp["nonterminals"].data_ptr(), inp["weights"].data_ptr(), C.f32(inp["kappa"]), C.f32(inp["gamma_n"]), B,
            loss.data_ptr(), dz.data_ptr(), T.data_ptr(), astar.data_ptr())
    L = lib()
    if inp.get("eps") is None:
        rc = L.rb_qr_dueling_loss_grad(*args, stream())
    else:
        rc = L.rb_qr_dueling_vt_loss_grad(*args, inp["eps"], stream())
    assert rc == 0, L.rb_last_error()
    return loss, dz, T, astar


def _guards(outs, B, M, K):
    for name, t, n in zip(("loss", "dz", "T", "astar"), outs, (B, M * B, B, K * B)):
        tail = t[n:]
        ok = bool((tail == -1).all()) if t.dtype == torch.int64 else bool(torch.isnan(tail).all())
        assert ok, f"{name}: written past its last row"


# (B, A, N, kappa, M, K, eps): every level of each range at least once, both R, both entries
CASES = [(32, 6, 51, 1.0, 2, 2, None), (1, 1, 2, 0.25, 1, 2, None), (33, 18, 65, 10.0, 2, 1, None),
         (512, 6, 64, 1.0, 2, 2, None), (35, 6, 128, 0.25, 3, 5, None), (42, 6, 51, 1.0, 8, 8, None),
         (33, 18, 128, 1.0, 2, 2, None), (32, 1, 65, 10.0, 3, 5, None),
         (32, 6, 51, 1.0, 2, 2, 1e-3), (33, 18, 65, 0.25, 3, 5, 0.0), (512, 6, 128, 10.0, 2, 1, 1e-3),
         (1, 6, 2, 1.0, 8, 8, 1e-3), (42, 1, 64, 1.0, 1, 2, 0.0)]


@pytest.mark.parametrize("case", CASES, ids=[f"B{c[0]}-A{c[1]}-N{c[2]}-k{c[3]:g}-M{c[4]}-K{c[5]}-e{c[6]}" for c in CASES])
def test_avg_loss_against_float64(case, tmp_path):
    B, A, N, kappa, M, K, eps = case
    inp = QD.make_inputs(B, A, N, kappa, 11 + B + N + 97 * M + K, M, K, eps)
    dev = C.to(inp, DEV)
    eager = run_avg(dev)
    _, outs, dot = graph_kernels(lambda: run_avg(dev), tmp_path / "avg.dot")
    want = f"k_qr_dueling_avg<{2 if N <= 64 else 4}>"
    assert variants_of(dot) == {want}, f"kernels launched {variants_of(dot)}, expected {want}"
    _guards(outs, B, M, K)
    _guards(eager, B, M, K)
    for name, a, b in zip(("loss", "dz", "T", "astar"), eager, outs):
        assert torch.equal(a, b) if name == "astar" else torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0)), \
            f"{name}: eager launch and graph replay differ"
    bare = run_avg(dev, with_outs=False)
    assert torch.equal(bare[0][:B], outs[0][:B]) and torch.equal(bare[1][:M * B], outs[1][:M * B]), \
        "theta_out / astar_out NULL changes the result"
    loss, dz, T, astar = outs[0][:B], outs[1][:M * B], outs[2][:B], outs[3][:K * B].view(K, B)

    assert bool(((astar >= 0) & (astar < A)).all()), "a* in range"
    T_ref, T_sc, _, ok = QD.target(dev, astar)
    assert ok, "a*_k within the arg-max's rounding"
    for k in range(K):
        assert bool(C.first_of_identical(QD.single(dev, 0, k), astar[k]).all()), "ties go to the first action"
    R.assert_within("Tbar", T, T_ref, T_sc, Q.TAU)
    (l_ref, l_sc), _, (dz_ref, dz_sc) = QD.loss_dz(dev, T)
    R.assert_within("loss", loss, l_ref, l_sc, Q.TAU)
    R.assert_within("dz", dz, dz_ref, dz_sc, Q.TAU)
    assert bool((loss >= 0).all())
    zero_w = dev["weights"] == 0
    assert bool((dz.view(M, B, -1)[:, zero_w] == 0).all()), "rows of weight 0 have an exactly zero gradient"


@pytest.mark.parametrize("B,A,N,eps", [(32, 6, 51, None), (35, 18, 128, None), (1, 1, 2, None), (512, 6, 51, None),
                                       (33, 6, 65, 1e-3), (32, 18, 64, 0.0)])
def test_one_copy_is_rb_qr_dueling_and_identical_copies_average_exactly(B, A, N, eps):
    inp = C.to(QD.make_inputs(B, A, N, 1.0, 3 + B + N, 1, 1, eps), DEV)
    single, avg = run_single(inp), run_avg(inp)
    torch.cuda.synchronize()
    for name, a, b in zip(("loss", "dz", "T", "astar"), single, avg):
        assert_bits_equal(cpu(b[:a.shape[0]]), cpu(a), f"M = K = 1: {name}")
    # x + x = 2x, 2x + x + x = 4x and the divisions by 2 and 4 are exact (a third copy, or eight, would round)
    for M, K in ((2, 2), (1, 4), (4, 1), (4, 4), (2, 1)):
        same = dict(inp, M=M, K=K, z_on=torch.cat([inp["z_on"][:B]] * M + [inp["z_on"][B:]] * K),
                    z_tg=torch.cat([inp["z_tg"]] * K))
        out = run_avg(same)
        torch.cuda.synchronize()
        assert_bits_equal(cpu(out[2][:B]), cpu(single[2]), f"identical copies M {M} K {K}: Tbar")
        assert_bits_equal(cpu(out[0][:B]), cpu(single[0]), f"identical copies M {M} K {K}: loss")
        assert_bits_equal(cpu(out[3][:K * B]), np.tile(cpu(single[3]), K), f"identical copies M {M} K {K}: a*")


@pytest.mark.parametrize("B,A,N,M,K,eps", [(33, 6, 51, 3, 5, None), (32, 18, 128, 2, 3, None), (35, 6, 65, 5, 3, 1e-3)])
def test_sums_run_in_copy_order(B, A, N, M, K, eps):
    """The definition's roundings, bitwise: a*_k and T_k are those of a one-copy launch on target copy k (M = K = 1 is
    rb_qr_dueling's, bitwise), Tbar = fl32(T_0 + T_1 + ...) in k order / K, and loss = fl32(loss_0 + loss_1 + ...) in j
    order / M with loss_j that of a launch on online copy j alone against the same K target copies."""
    inp = C.to(QD.make_inputs(B, A, N, 1.0, 7 + B + N, M, K, eps), DEV)

    def sub(js, ks):
        return dict(inp, M=len(js), K=len(ks), z_on=torch.cat([inp["z_on"][j * B:(j + 1) * B] for j in js] +
                                                              [inp["z_on"][(M + k) * B:(M + k + 1) * B] for k in ks]),
                    z_tg=torch.cat([inp["z_tg"][k * B:(k + 1) * B] for k in ks]))
    full = [cpu(t) for t in run_avg(inp)]
    ones = [[cpu(t) for t in run_avg(sub([0], [k]))] for k in range(K)]
    per_j = [[cpu(t) for t in run_avg(sub([j], range(K)))] for j in range(M)]
    torch.cuda.synchronize()
    acc = ones[0][2][:B].copy()
    for k in range(1, K):
        acc = (acc + ones[k][2][:B]).astype(np.float32)
    assert_bits_equal(full[2][:B], (acc / np.float32(K)).astype(np.float32), "Tbar = (sum_k T_k in k order) / K")
    assert_bits_equal(full[3][:K * B], np.concatenate([o[3][:B] for o in ones]), "a*_k")
    for j in range(M):
        assert_bits_equal(per_j[j][2][:B], full[2][:B], f"copy {j} alone sees the same Tbar")
    acc = per_j[0][0][:B].copy()
    for j in range(1, M):
        acc = (acc + per_j[j][0][:B]).astype(np.float32)
    assert_bits_equal(full[0][:B], (acc / np.float32(M)).astype(np.float32), "loss = (sum_j loss_j in j order) / M")


@pytest.mark.parametrize("vt", [False, True], ids=["plain", "vt"])
def test_oversize_is_refused_and_writes_nothing(vt):
    from rainbow_b200 import _lib
    B, A, N, M, K = 4, 64, 128, 8, 8     # (M + 2K) (N + A N) floats = 780 KB of shared memory
    inp = C.to(QD.make_inputs(B, 2, N, 1.0, 5, 1, 1, 1e-3 if vt else None), DEV)
    z_on = torch.zeros((M + K) * B, N + A * N, device=DEV)
    z_tg = torch.zeros(K * B, N + A * N, device=DEV)
    outs = [torch.full((B,), NAN, device=DEV), torch.full((M * B, N + A * N), NAN, device=DEV),
            torch.full((B, N), NAN, device=DEV), torch.full((K * B,), -1, dtype=torch.int64, device=DEV)]
    args = (z_on.data_ptr(), z_tg.data_ptr(), A, N, inp["actions"].data_ptr(), inp["returns"].data_ptr(),
            inp["nonterminals"].data_ptr(), inp["weights"].data_ptr(), 1.0, 0.97, B, M, K) + tuple(t.data_ptr() for t in outs)
    L = lib()
    rc = L.rb_qr_dueling_avg_vt_loss_grad(*args, 1e-3, stream()) if vt else L.rb_qr_dueling_avg_loss_grad(*args, stream())
    assert rc == -34 and b"too large" in L.rb_last_error()
    torch.cuda.synchronize()
    assert all(bool(torch.isnan(t).all()) for t in outs[:3]) and bool((outs[3] == -1).all()), "a refused call writes nothing"
    with pytest.raises(_lib.RainbowB200Error):
        from rainbow_b200.agent import qr_dueling_avg_loss_grad
        qr_dueling_avg_loss_grad(z_on, z_tg, A, N, inp["actions"], inp["returns"], inp["nonterminals"], inp["weights"],
                                 1.0, 0.97, M, K)


# ---- the learner -----------------------------------------------------------------------------------------------------------
QRD = dict(distribution="quantile", quantile_kappa=1.0, quantile_average_copies=True)
DRQ = dict(QRD, augment_shift=4, augment_intensity=0.05, augment_m=2, augment_k=2)


def _agent(seed=5, **kw):
    from rainbow_b200.agent import Agent
    torch.manual_seed(seed)
    return Agent(make_args(**kw), FakeEnv(6))


def _memory(**args):
    mem, _ = synthetic_ring(CAP, seed=3, args=args)
    mem.seed = 99
    return mem


def test_identical_copies_equal_a_plain_agent():
    """Pad 0, intensity 0, M = K = 2: two identical copies, so Tbar = (T + T) / 2 and loss = (l + l) / 2 are exact and each
    copy's gradient is half the plain one (w / 2B); the backward sums the two halves in another order."""
    for kw in (dict(), dict(architecture="data-efficient", hidden_size=256, multi_step=20)):
        dup = _agent(augment_m=2, augment_k=2, learn_stats=8, cuda_graph=False, **QRD, **kw)
        plain = _agent(learn_stats=8, cuda_graph=False, **QRD, **kw)
        assert dup.quantile_average_copies and not plain.quantile_average_copies
        mem_kw = {k: v for k, v in kw.items() if k == "multi_step"}
        md, mp = _memory(**mem_kw), _memory(**mem_kw)
        for ag, mem in ((dup, md), (plain, mp)):
            ag.reset_noise()
            ag.learn(mem)
        torch.cuda.synchronize()
        assert_bits_equal(cpu(dup.last_loss), cpu(plain.last_loss), "loss")
        assert_bits_equal(cpu(dup._stats["last"]["m"]), cpu(plain._stats["last"]["m"]), "Tbar")
        assert_bits_equal(cpu(md.transitions.tree), cpu(mp.transitions.tree), "priorities")
        gd, gp = dup.optimiser.flat_grad.double(), plain.optimiser.flat_grad.double()
        assert float((gd - gp).abs().max()) <= 5e-7 * float(gp.abs().max())


def test_graph_replay_equals_eager():
    ga, ea = _agent(**DRQ), _agent(cuda_graph=False, **DRQ)
    gm, em = _memory(), _memory()
    for step in range(7):
        for ag, mem in ((ga, gm), (ea, em)):
            ag.reset_noise()
            ag.learn(mem)
        assert_bits_equal(cpu(ga.last_loss), cpu(ea.last_loss), f"loss of update {step}")
    assert ga._graphs and not ea._graphs
    torch.cuda.synchronize()
    for k in ("flat_param", "exp_avg", "exp_avg_sq"):
        assert_bits_equal(cpu(getattr(ga.optimiser, k)), cpu(getattr(ea.optimiser, k)), k)
    assert_bits_equal(cpu(gm.transitions.tree), cpu(em.transitions.tree), "tree")


def test_update_graph_nodes(tmp_path, monkeypatch):
    names = {}
    intensity = dict(augment_shift=4, augment_intensity=0.05)
    for tag, kw in (("qr", dict(distribution="quantile")), ("qr-switch", dict(QRD, augment_m=1, augment_k=1)),
                    ("qr-intensity", dict(distribution="quantile", **intensity)), ("qr-drq", DRQ)):
        names[tag] = update_graph(_agent(**kw), _memory(), tmp_path / f"{tag}.dot", monkeypatch)
    assert names["qr-switch"] == names["qr"], "the switch at M = K = 1 leaves the quantile update graph as it is"
    assert "k_qr_dueling_avg" not in names["qr"] and "k_qr_dueling" in names["qr"]
    drq = names["qr-drq"]
    assert drq.count("k_qr_dueling_avg") == 1 and "k_qr_dueling" not in drq
    own = lambda ks: [k for k in ks if k.startswith("k_")]
    want = []
    for k in own(names["qr-intensity"]):
        want += {"k_qr_dueling": ["k_qr_dueling_avg"], "k_head_bwd1": ["k_head_bwd1_wgrad", "k_head_bwd1_dx"]}.get(k, [k])
    assert own(drq) == want


def test_resume_equals_never_stopping_and_a_mismatched_switch_is_refused(tmp_path):
    from test_gpu_checkpoint import _agent as ck_agent
    from test_gpu_checkpoint import _assert_same, _before_update, _fresh_memory, _refused, _state, _update
    from test_gpu_checkpoint import _memory as ck_memory
    total, save_at = 12, 5
    ag, mem = ck_agent(**DRQ), ck_memory()
    losses = []
    for step in range(total):
        _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    run_a = _state(ag, mem, losses)

    ag, mem = ck_agent(**DRQ), ck_memory()
    losses = []
    for step in range(save_at):
        _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _before_update(ag, mem, save_at, True)
    ag.save_checkpoint(str(tmp_path / "ck"), mem)
    hp = json.load(open(tmp_path / "ck" / "rank0" / "manifest.json"))["hyper_parameters"]
    assert hp["quantile_average_copies"] is True and (hp["distribution"], hp["augment_m"], hp["augment_k"]) == \
        ("quantile", 2, 2)
    ag, mem = ck_agent(seed=77, **DRQ), _fresh_memory()
    ag.load_checkpoint(str(tmp_path / "ck"), mem)
    for step in range(save_at, total):
        if step > save_at:
            _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _assert_same(run_a, _state(ag, mem, losses))

    # a quantile learner without copies does not record the switch, and neither side loads the other
    plain = ck_agent(**dict(QRD, augment_shift=4, augment_intensity=0.05))
    plain.save_checkpoint(str(tmp_path / "plain"))
    hp = json.load(open(tmp_path / "plain" / "rank0" / "manifest.json"))["hyper_parameters"]
    assert "quantile_average_copies" not in hp
    ag.save_checkpoint(str(tmp_path / "drq"))
    _refused(ck_agent(seed=8, **DRQ), None, str(tmp_path / "plain"), match="quantile_average_copies")
    _refused(plain, None, str(tmp_path / "drq"), match="quantile_average_copies")


def test_learn_stats_hold_the_averaged_loss_and_tbar():
    ag = _agent(learn_stats=8, **DRQ)
    mem = _memory()
    for _ in range(3):
        ag.reset_noise()
        ag.learn(mem)
    torch.cuda.synchronize()
    rec = ag.learn_stats()
    assert len(rec["loss_mean"]) == 3
    loss = cpu(ag.last_loss).astype(np.float64)
    assert rec["loss_mean"][-1] == pytest.approx(float(loss.mean()), rel=1e-6)
    assert rec["loss_max"][-1] == cpu(ag.last_loss).max()
    T = cpu(ag._stats["last"]["m"]).astype(np.float64)
    assert rec["target_mean"][-1] == pytest.approx(float(T.mean()), rel=1e-5, abs=1e-6)


def test_acting_is_not_augmented():
    kw = dict(architecture="data-efficient", hidden_size=64)
    aug, plain = _agent(**DRQ, **kw), _agent(**QRD, **kw)
    val, _ = synthetic_ring(256, seed=4)
    states = val.iter_states(0, 8)
    for i in range(4):
        assert aug.act(states[i]) == plain.act(states[i])
    assert aug.evaluate_q_memory(val) == plain.evaluate_q_memory(val)


def test_library_head_with_copies_is_refused():
    from rainbow_b200 import RainbowB200Error
    kw = dict(architecture="data-efficient", hidden_size=64)
    for bad in (dict(fused_head=False), dict(batch_size=512)):
        refused, mem = _agent(cuda_graph=False, **DRQ, **bad, **kw), _memory()
        counter, tree = mem._rng_counter.clone(), mem.transitions.tree.clone()
        with pytest.raises(RainbowB200Error, match="fused head"):
            refused.learn(mem)
        assert torch.equal(mem._rng_counter, counter) and torch.equal(mem.transitions.tree, tree), "nothing sampled"
        assert int(refused.optimiser.step_count.item()) == 0


@pytest.mark.parametrize("eps", [1e-3, 0.0])
def test_value_rescaling_with_copies_on_the_learners_own_rows(eps, monkeypatch):
    """One eager fused update with M = K = 2, shift 4, intensity 0.05 and value rescaling: the loss kernel's own inputs
    (the heads' z rows and the batch) are captured, and its loss, Tbar (the statistics rows) and dz held to
    tests/qr_drq_ref.py's vt_ref-based reference; the priorities are fl32(sqrt(loss)) bitwise."""
    import rainbow_b200.agent as agent_mod
    seen = {}
    orig = agent_mod.qr_dueling_avg_loss_grad

    def spy(z_online, z_target, actions_n, atoms, actions, returns, nonterminals, weights, kappa, gamma_n, M, K, **kw):
        astar = torch.full((K, actions.shape[0]), -1, dtype=torch.int64, device=actions.device)
        kw = dict(kw, astar_out=astar)   # an optional output: the results do not depend on it
        loss, dz = orig(z_online, z_target, actions_n, atoms, actions, returns, nonterminals, weights, kappa, gamma_n, M, K,
                        **kw)
        seen.update(z_on=z_online.clone(), z_tg=z_target.clone(), actions=actions.clone(), returns=returns.clone(),
                    nonterminals=nonterminals.clone(), weights=weights.clone(), kappa=kappa, gamma_n=gamma_n, M=M, K=K,
                    eps=kw["eps"], T=kw["theta_out"], astar=astar, loss=loss, dz=dz)
        return loss, dz
    monkeypatch.setattr(agent_mod, "qr_dueling_avg_loss_grad", spy)
    ag = _agent(cuda_graph=False, learn_stats=4, value_transform="rescale", value_transform_eps=eps, **DRQ)
    mem = _memory()
    for _ in range(2):
        ag.reset_noise()
        ag.learn(mem)
    torch.cuda.synchronize()
    assert seen["eps"] == float(np.float32(eps)) and (seen["M"], seen["K"]) == (2, 2)   # the fp32 the kernels take
    B, A, N = ag.batch_size, ag.action_space, ag.atoms
    inp = dict(entry="dueling", B=B, A=A, Z=N, M=2, K=2, kappa=seen["kappa"], gamma_n=seen["gamma_n"], eps=seen["eps"],
               z_on=seen["z_on"][:4 * B], z_tg=seen["z_tg"][:2 * B], actions=seen["actions"], returns=seen["returns"],
               nonterminals=seen["nonterminals"], weights=seen["weights"])
    assert not torch.equal(inp["z_on"][:B], inp["z_on"][B:2 * B]), "the copies differ"
    T_ref, T_sc, _, ok = QD.target(inp, seen["astar"])
    assert ok, "a*_k within the arg-max's rounding"
    R.assert_within("Tbar", seen["T"], T_ref, T_sc, Q.TAU)
    (l_ref, l_sc), _, (dz_ref, dz_sc) = QD.loss_dz(inp, seen["T"])
    R.assert_within("loss", seen["loss"], l_ref, l_sc, Q.TAU)
    R.assert_within("dz", seen["dz"], dz_ref, dz_sc, Q.TAU)
    assert torch.equal(seen["loss"], ag.last_loss)
    tidx, got = cpu(mem._last.tree_idx), cpu(ag.last_loss)
    last = np.array([i for i in range(len(tidx)) if tidx[i] not in tidx[i + 1:]])
    assert_bits_equal(cpu(mem.transitions.tree)[tidx[last]], np.sqrt(got)[last], "priorities")


# ---- whole updates against float64 -----------------------------------------------------------------------------------------
QR_DRQ_CASES = [
    _row("quantile", "drq", "fixed", "adam", "polyak", "on", "on", "off", 1, "fused", "c-h512", "flushed"),
    _row("quantile", "drq", "annealed", "adamw", "hard", "off", "on", "on", 32, "fused", "de-h256", "pending"),
    _row("quantile", "drq", "annealed", "adam", "hard", "on", "off", "on", 33, "fused", "c-h64", "flushed"),
    _row("quantile", "drq", "fixed", "adamw", "polyak", "off", "off", "off", 64, "fused", "de-h256", "pending"),
]


@pytest.mark.parametrize("c", QR_DRQ_CASES, ids=[case_id(c) for c in QR_DRQ_CASES])
def test_update_trajectory_against_float64(c, tmp_path, monkeypatch):
    """test_gpu_update_f64's trajectory check as it stands, with the switch set and k_qr_dueling_avg the loss node."""
    kwargs, kernels = TU.agent_kwargs, TU._expected_kernels

    def expected(case, ag):
        gather, loss, bwd = kernels(case, ag)
        return gather, "k_qr_dueling_avg" if loss == "k_qr_dueling" else loss, bwd
    monkeypatch.setattr(TU, "agent_kwargs", lambda case: dict(kwargs(case), quantile_average_copies=True))
    monkeypatch.setattr(TU, "_expected_kernels", expected)
    TU.test_update_trajectory_against_float64(c, tmp_path, monkeypatch)
