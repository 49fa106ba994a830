"""Munchausen targets under the quantile loss on the GPU (rb_qr_dueling_munchausen_loss_grad -> k_qr_dueling_munchausen<R>,
rb_qr_munchausen_loss_grad -> k_qr_munchausen<R>, args.munchausen).

* The kernels: T, b, the loss and every dz / grad element against tests/munchausen_ref.py (|err| <= qr_ref.TAU x scale)
  over N 51 / 128 (R = 2 / 4), A 3 / 6 / 18, B 1 / 32 / 512, tau 0.03 / 1 and alpha 0 / 0.9, with qr_ref's row kinds
  (terminals, weight 0) and rows whose target means spread by 3 per action (the clip binds there).  Outputs are prefilled
  with NaN and guard rows past each must stay untouched; the template variant is read from a captured graph's nodes; the
  graph replay, the eager launch and a launch without the optional outputs agree bitwise.  T is the definition's fp32
  operation order bitwise (an emulation with separately rounded torch operations).  A refused call writes nothing.
* The learner: the update graph is the quantile graph with k_qr_dueling_munchausen in k_qr_dueling's place and the same
  launch count, the online head on B rows and the target head on 2B; graph replays equal eager updates; resume equals
  never stopping and a mismatched checkpoint is refused in both directions; the annealed horizon is the fixed horizon
  bitwise; acting is unchanged; the statistics hold T.  On the learner's own head rows, one update's loss, T and dz (or
  grad) against the reference, for the fused head at B 32 and 64, C3, the library head and every composable switch.
* Whole updates: tests/test_gpu_update_f64.py's trajectory check, unchanged, over the same five kinds of case, against
  tests/munchausen_update_ref.py (gradients per element, the optimiser step, gather, target, resets, ReDo, statistics)."""
import json
import re

import numpy as np
import pytest
import torch

import c51_ref as C
import head_ref as R
import munchausen_ref as MR
import qr_ref as Q
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


def _p(t):
    return None if t is None else t.data_ptr()


def run(inp, with_outs=True):
    """One launch of inp's entry into NaN-prefilled outputs with GUARD rows past each: (loss, dz or grad, T, b)."""
    B, A, N = inp["B"], inp["A"], inp["Z"]
    loss = torch.full((B + GUARD,), NAN, device=DEV)
    T = torch.full((B + GUARD, N), NAN, device=DEV) if with_outs else None
    b = torch.full((B + GUARD,), NAN, device=DEV) if with_outs else None
    par = (C.f32(inp["kappa"]), C.f32(inp["gamma_n"]), inp["alpha"], inp["tau"], inp["clip"])
    common = (inp["actions"].data_ptr(), inp["returns"].data_ptr(), inp["nonterminals"].data_ptr(),
              inp["weights"].data_ptr())
    L = lib()
    if inp["entry"] == "plain":
        g = torch.full((B + GUARD, A, N), NAN, device=DEV)
        rc = L.rb_qr_munchausen_loss_grad(inp["q_on_s"].data_ptr(), inp["q_tg_s"].data_ptr(), inp["q_tg_ns"].data_ptr(),
                                          *common, *par, B, A, N, loss.data_ptr(), g.data_ptr(), _p(T), _p(b), stream())
    else:
        g = torch.full((B + GUARD, N + A * N), NAN, device=DEV)
        rc = L.rb_qr_dueling_munchausen_loss_grad(inp["z_on"].data_ptr(), inp["z_tg"].data_ptr(), A, N, *common, *par, B,
                                                  loss.data_ptr(), g.data_ptr(), _p(T), _p(b), stream())
    assert rc == 0, L.rb_last_error()
    return loss, g, T, b


def _guards(outs, B):
    for name, t in zip(("loss", "grad", "T", "b"), outs):
        if t is not None:
            assert bool(torch.isnan(t[B:]).all()), f"{name}: written past its last row"


_K = re.compile(r"k_qr(_dueling)?_munchausen(?:<\s*(\d)\s*>|ILi(\d)E)")


def variants_of(dot):
    return {f"k_qr{d}_munchausen<{a or b}>" for d, a, b in _K.findall(dot)}


# (entry, B, A, N, tau, alpha): N on both sides of the R switch; each N meets every B x tau x alpha level, each A twice
_LEVELS = [(32, 0.03, 0.9), (512, 1.0, 0.0), (1, 1.0, 0.9), (32, 1.0, 0.0), (512, 0.03, 0.9), (1, 0.03, 0.0)]
GRID = [(e, *_LEVELS[j][:1], A, N, *_LEVELS[j][1:])
        for e in ("dueling", "plain")
        for k, (N, A) in enumerate(((51, 3), (51, 6), (51, 18), (128, 3), (128, 6), (128, 18)))
        for j in (k, (k + 3) % 6)]


@pytest.mark.parametrize("case", GRID, ids=[f"{c[0]}-B{c[1]}-A{c[2]}-N{c[3]}-t{c[4]:g}-a{c[5]:g}" for c in GRID])
def test_loss_against_float64(case, tmp_path):
    entry, B, A, N, tau, alpha = case
    inp = C.to(MR.make_inputs(entry, B, A, N, 1.0, 31 + B + N + A, alpha=alpha, tau=tau), DEV)
    eager = run(inp)
    _, outs, dot = graph_kernels(lambda: run(inp), tmp_path / "m.dot")
    want = f"k_qr{'_dueling' if entry == 'dueling' else ''}_munchausen<{2 if N <= 64 else 4}>"
    assert variants_of(dot) == {want}, f"kernels launched {variants_of(dot)}, expected {want}"
    _guards(outs, B)
    _guards(eager, B)
    for name, a, b in zip(("loss", "grad", "T", "b"), eager, outs):
        assert torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0)), f"{name}: eager launch and graph replay differ"
    bare = run(inp, with_outs=False)
    assert torch.equal(bare[0][:B], outs[0][:B]) and torch.equal(bare[1][:B], outs[1][:B]), \
        "theta_out / bonus_out NULL changes the result"
    loss, g, T, b = (t[:B] for t in outs)

    T_ref, T_sc, b_ref, b_sc, near = MR.targets(inp)
    R.assert_within("b", b, b_ref, b_sc, Q.TAU)
    R.assert_within("T", T, T_ref, T_sc, Q.TAU)
    if alpha == 0.0:
        assert bool((b == 0).all())
    clipped = (b_ref == inp["alpha"] * inp["clip"]) & ~near
    assert torch.equal(b[clipped], torch.full_like(b[clipped], C.f32(inp["alpha"] * np.float32(inp["clip"])))), \
        "where the clip binds b is fl32(alpha l0)"
    (l_ref, l_sc), (g_ref, g_sc) = MR.loss_grad(inp, T)
    R.assert_within("loss", loss, l_ref, l_sc, Q.TAU)
    if entry == "dueling":
        d_ref, d_sc = MR.dz(inp, g_ref, g_sc)
    else:
        d_ref, d_sc = MR.grad_rows(inp, g_ref, g_sc)
    R.assert_within("grad", g, d_ref, d_sc, Q.TAU)
    assert bool((loss >= 0).all())
    zero_w = inp["weights"] == 0
    assert bool((g[zero_w] == 0).all()), "rows of weight 0 have an exactly zero gradient"


def test_grid_has_clipped_terminal_and_spread_rows():
    for entry, B, A, N, tau, alpha in GRID:
        if B < 32:
            continue
        inp = MR.make_inputs(entry, B, A, N, 1.0, 31 + B + N + A, alpha=alpha, tau=tau)
        _, _, b, _, _ = MR.targets(inp)
        lam = b == inp["alpha"] * inp["clip"]
        if alpha > 0:
            assert bool(lam.any()) and bool((~lam).any()), (entry, B, A, N, tau)
        assert bool((inp["nonterminals"] == 0).any())


def _fp32_target(q_s, q_ns, theta_ns, acts, r, nt, gamma_n, alpha, tau, l0):
    """T [B][N] and b [B] with the kernel's operation order in separately rounded fp32 torch operations: qr_row_mean's
    lane sums and butterfly, then the stage; q_s, q_ns, theta_ns [B][A][N] are the target's per-action quantile rows."""
    B, A, N = q_ns.shape
    Rr = -(-N // 32)

    def mean(q):
        x = torch.zeros(B, A, 32 * Rr, device=DEV)
        x[:, :, :N] = q
        p = torch.zeros(B, A, 32, device=DEV)
        for r in range(Rr):
            p = p + x[:, :, 32 * r:32 * (r + 1)]
        for o in (16, 8, 4, 2, 1):
            p = p + p[:, :, torch.arange(32, device=DEV) ^ o]
        return p[:, :, 0] / torch.full_like(p[:, :, 0], float(N))

    def stage(q):
        m = q.max(1, keepdim=True).values
        d = q - m
        e = torch.exp(d / torch.full_like(d, tau))
        S = torch.zeros(B, 1, device=DEV)
        for a in range(A):
            S = S + e[:, a:a + 1]
        tl = torch.log(S) * tau
        return e / S, d - tl

    pi_s, l_s = stage(mean(q_s))
    b = torch.maximum(l_s[torch.arange(B), acts], torch.full((B,), l0, device=DEV)) * alpha
    pi, l = stage(mean(q_ns))
    c = torch.zeros(B, N, device=DEV)
    for a in range(A):
        c = c + pi[:, a:a + 1] * (theta_ns[:, a] - l[:, a:a + 1])
    sc = nt.view(-1) * gamma_n
    return (r + b).unsqueeze(1) + sc.unsqueeze(1) * c, b


@pytest.mark.parametrize("entry,B,A,N,tau", [("plain", 64, 6, 51, 0.03), ("plain", 33, 18, 128, 1.0),
                                             ("dueling", 64, 6, 51, 0.03), ("dueling", 35, 3, 128, 1.0)])
def test_sums_run_in_the_stated_order(entry, B, A, N, tau):
    inp = C.to(MR.make_inputs(entry, B, A, N, 1.0, 5 + B, tau=tau), DEV)
    _, _, T, b = run(inp)
    if entry == "plain":
        rows = inp["q_tg_s"], inp["q_tg_ns"]
    else:
        def dq(z):     # the dueling combination in the kernel's order: (v + adv) - (sum_a adv in order) / A
            v, adv = z[:, :N].unsqueeze(1), z[:, N:].view(B, A, N)
            acc = torch.zeros(B, 1, N, device=DEV)
            for a in range(A):
                acc = acc + adv[:, a:a + 1]
            return (v + adv) - acc / torch.full_like(acc, float(A))
        rows = dq(inp["z_tg"][:B]), dq(inp["z_tg"][B:])
    want_T, want_b = _fp32_target(rows[0], rows[1], rows[1], inp["actions"], inp["returns"], inp["nonterminals"],
                                  C.f32(inp["gamma_n"]), inp["alpha"], inp["tau"], inp["clip"])
    torch.cuda.synchronize()
    assert_bits_equal(cpu(b[:B]), cpu(want_b), "b")
    assert_bits_equal(cpu(T[:B]), cpu(want_T), "T")


@pytest.mark.parametrize("entry", ["dueling", "plain"])
def test_refused_calls_write_nothing(entry):
    from rainbow_b200.agent import qr_dueling_munchausen_loss_grad
    inp = C.to(MR.make_inputs(entry, 8, 6, 51, 1.0, 3), DEV)
    for change in (dict(alpha=NAN), dict(tau=0.0), dict(clip=0.0)):
        bad = dict(inp, **change)
        loss, g = torch.full((8,), NAN, device=DEV), torch.full((8, 7 * 51), NAN, device=DEV)
        T, b = torch.full((8, 51), NAN, device=DEV), torch.full((8,), NAN, device=DEV)
        par = (1.0, 0.97, bad["alpha"], bad["tau"], bad["clip"])
        common = (bad["actions"].data_ptr(), bad["returns"].data_ptr(), bad["nonterminals"].data_ptr(),
                  bad["weights"].data_ptr())
        if entry == "plain":
            rc = lib().rb_qr_munchausen_loss_grad(bad["q_on_s"].data_ptr(), bad["q_tg_s"].data_ptr(),
                                                  bad["q_tg_ns"].data_ptr(), *common, *par, 8, 6, 51, loss.data_ptr(),
                                                  g.data_ptr(), T.data_ptr(), b.data_ptr(), stream())
        else:
            rc = lib().rb_qr_dueling_munchausen_loss_grad(bad["z_on"].data_ptr(), bad["z_tg"].data_ptr(), 6, 51, *common,
                                                          *par, 8, loss.data_ptr(), g.data_ptr(), T.data_ptr(),
                                                          b.data_ptr(), stream())
        assert rc == -22
        torch.cuda.synchronize()
        assert all(bool(torch.isnan(t).all()) for t in (loss, g, T, b)), "a refused call writes nothing"
    from rainbow_b200 import _lib
    z = torch.zeros(8, 201 * 128, device=DEV)
    with pytest.raises(_lib.RainbowB200Error, match="too large"):
        qr_dueling_munchausen_loss_grad(z, torch.cat([z, z]), 200, 128, inp["actions"], inp["returns"],
                                        inp["nonterminals"], inp["weights"], 1.0, 0.97, 0.9, 0.03, -1.0)


# ---- the learner -----------------------------------------------------------------------------------------------------------
MUNCH = dict(distribution="quantile", munchausen=True)
ALL = dict(MUNCH, augment_shift=4, augment_intensity=0.05, target_tau=0.005, reset_interval=5, redo_interval=3,
           weight_decay=0.1, reset_optimizer=True, learn_stats=8, anneal_steps=6, multi_step_start=10, discount_start=0.97,
           multi_step=3, discount=0.997)
MEM_ALL = dict(anneal_steps=6, multi_step_start=10, discount_start=0.97, multi_step=3, discount=0.997)


def _agent(seed=5, **kw):
    from rainbow_b200.agent import Agent
    torch.manual_seed(seed)
    return Agent(make_args(**kw), FakeEnv(6))


def _memory(**args):
    mem, _ = synthetic_ring(CAP, seed=3, args=args)
    mem.seed = 99
    return mem


def test_update_graph_nodes(tmp_path, monkeypatch):
    names = {}
    ags = {}
    for tag, kw in (("qr", dict(distribution="quantile")), ("off", dict(distribution="quantile", munchausen=False)),
                    ("m", MUNCH)):
        ags[tag] = _agent(**kw)
        names[tag] = update_graph(ags[tag], _memory(), tmp_path / f"{tag}.dot", monkeypatch)
    assert names["off"] == names["qr"], "munchausen = False leaves the update graph as it is"
    own = lambda ks: [k for k in ks if k.startswith("k_")]
    m = own(names["m"])
    assert m.count("k_qr_dueling_munchausen") == 1 and "k_qr_dueling" not in m
    assert m == [{"k_qr_dueling": "k_qr_dueling_munchausen"}.get(k, k) for k in own(names["qr"])]
    assert len(names["m"]) == len(names["qr"]), "the same node count"
    B = ags["m"].batch_size
    assert set(ags["m"].online_net.head()._scratch) == {B}, "the online head runs on s only"
    assert set(ags["m"].target_net.head()._scratch) == {2 * B}, "the target head runs on [s; s']"
    assert set(ags["qr"].online_net.head()._scratch) == {2 * B} and set(ags["qr"].target_net.head()._scratch) == {B}


def test_graph_replay_equals_eager():
    kw = dict(ALL)
    ga, ea = _agent(**kw), _agent(cuda_graph=False, **kw)
    gm, em = _memory(**MEM_ALL), _memory(**MEM_ALL)
    for step in range(8):
        for ag, mem in ((ga, gm), (ea, em)):
            ag.reset_noise()
            ag.learn(mem)
        assert_bits_equal(cpu(ga.last_loss), cpu(ea.last_loss), f"loss of update {step}")
    assert ga._graphs and not ea._graphs
    torch.cuda.synchronize()
    for k in ("flat_param", "exp_avg", "exp_avg_sq"):
        assert_bits_equal(cpu(getattr(ga.optimiser, k)), cpu(getattr(ea.optimiser, k)), k)
    assert_bits_equal(cpu(gm.transitions.tree), cpu(em.transitions.tree), "tree")
    assert_bits_equal(cpu(ga.target_flat), cpu(ea.target_flat), "target")


def test_resume_equals_never_stopping_and_a_mismatch_is_refused(tmp_path):
    from test_gpu_checkpoint import _agent as ck_agent
    from test_gpu_checkpoint import _assert_same, _before_update, _fresh_memory, _refused, _state, _update
    from test_gpu_checkpoint import _memory as ck_memory
    kw = dict(MUNCH, augment_shift=4, munchausen_alpha=0.8)
    total, save_at = 10, 4
    ag, mem = ck_agent(**kw), ck_memory()
    losses = []
    for step in range(total):
        _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    run_a = _state(ag, mem, losses)

    ag, mem = ck_agent(**kw), ck_memory()
    losses = []
    for step in range(save_at):
        _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _before_update(ag, mem, save_at, True)
    ag.save_checkpoint(str(tmp_path / "ck"), mem)
    hp = json.load(open(tmp_path / "ck" / "rank0" / "manifest.json"))["hyper_parameters"]
    assert (hp["munchausen_alpha"], hp["munchausen_temperature"], hp["munchausen_clip"]) == ag.munchausen
    ag, mem = ck_agent(seed=77, **kw), _fresh_memory()
    ag.load_checkpoint(str(tmp_path / "ck"), mem)
    for step in range(save_at, total):
        if step > save_at:
            _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _assert_same(run_a, _state(ag, mem, losses))

    plain = ck_agent(distribution="quantile", augment_shift=4)
    plain.save_checkpoint(str(tmp_path / "plain"))
    hp = json.load(open(tmp_path / "plain" / "rank0" / "manifest.json"))["hyper_parameters"]
    assert not any(k.startswith("munchausen") for k in hp)
    ag.save_checkpoint(str(tmp_path / "m"))
    _refused(ck_agent(seed=8, **kw), None, str(tmp_path / "plain"), match="munchausen")
    _refused(plain, None, str(tmp_path / "m"), match="munchausen")
    _refused(ck_agent(seed=8, **dict(kw, munchausen_temperature=1.0)), None, str(tmp_path / "m"), match="munchausen")


@pytest.mark.parametrize("case", ["fused-pending", "batch64", "c3", "library-head"])
def test_annealed_horizon_is_the_fixed_horizon(case, monkeypatch):
    """test_gpu_horizon's check as it stands, with both agents built under Munchausen."""
    import test_gpu_horizon as TH
    orig = TH._agent
    monkeypatch.setattr(TH, "_agent", lambda seed=5, **kw: orig(seed, **dict(kw, **MUNCH)))
    TH.test_annealed_update_is_the_plain_update_at_its_horizon(case)


def test_acting_is_unchanged():
    kw = dict(architecture="data-efficient", hidden_size=64, distribution="quantile")
    m, plain = _agent(munchausen=True, **kw), _agent(**kw)
    val, _ = synthetic_ring(256, seed=4)
    states = val.iter_states(0, 8)
    for i in range(4):
        assert m.act(states[i]) == plain.act(states[i])
    assert m.evaluate_q_memory(val) == plain.evaluate_q_memory(val)


def test_learn_stats_hold_t():
    ag = _agent(learn_stats=8, **MUNCH)
    mem = _memory()
    for _ in range(3):
        ag.reset_noise()
        ag.learn(mem)
    torch.cuda.synchronize()
    rec = ag.learn_stats()
    assert len(rec["loss_mean"]) == 3
    loss = cpu(ag.last_loss).astype(np.float64)
    assert rec["loss_mean"][-1] == pytest.approx(float(loss.mean()), rel=1e-6)
    T = cpu(ag._stats["last"]["m"]).astype(np.float64)
    assert np.isfinite(T).all()
    assert rec["target_mean"][-1] == pytest.approx(float(T.mean()), rel=1e-5, abs=1e-6)


# ---- one update on the learner's own rows ------------------------------------------------------------------------------------
OWN_CASES = {
    "fused-b32": (dict(), {}),
    "fused-b64": (dict(batch_size=64), {}),
    "c3": (dict(architecture="data-efficient", hidden_size=256, multi_step=20), dict(multi_step=20)),
    "library-head": (dict(fused_head=False), {}),
    "all-switches": (ALL, MEM_ALL),
}


@pytest.mark.parametrize("case", list(OWN_CASES))
def test_update_on_the_learners_own_rows(case, monkeypatch):
    """Eager updates whose loss kernel's own inputs -- the heads' rows and the batch -- are captured: the loss, T (the
    statistics rows), dz / grad held to tests/munchausen_ref.py; the priorities are fl32(sqrt(loss)) bitwise.  In the first
    update of the unaugmented cases the target rows the kernel read are the target net's forward of the batch's [s; s'],
    and the online rows the online net's forward of s with the parameters the update started from."""
    import rainbow_b200.agent as agent_mod
    kw, mem_kw = OWN_CASES[case]
    fused = case != "library-head"
    name = "qr_dueling_munchausen_loss_grad" if fused else "qr_munchausen_loss_grad"
    seen = {}
    orig = getattr(agent_mod, name)

    def spy(*a, **k):
        b = torch.full((a[4 if fused else 3].shape[0],), NAN, device=DEV)
        out = orig(*a, **dict(k, bonus_out=b))
        seen.update(args=[x.clone() if isinstance(x, torch.Tensor) else x for x in a], T=k["theta_out"].clone(), b=b,
                    loss=out[0].clone(), grad=out[1].clone())
        return out
    monkeypatch.setattr(agent_mod, name, spy)
    ag = _agent(cuda_graph=False, **{"learn_stats": 4, **MUNCH, **kw})
    assert ag.munchausen is not None
    assert ag._fused_path(ag.batch_size) == fused
    mem = _memory(**mem_kw)
    for u in range(3):
        ag.reset_noise()
        p_before = ag.optimiser.flat_param.clone()
        ag.learn(mem)
        torch.cuda.synchronize()
        a = seen["args"]
        B, A, N = ag.batch_size, ag.action_space, ag.atoms
        alpha, tau, clip = ag.munchausen
        if fused:
            inp = dict(entry="dueling", B=B, A=A, Z=N, z_on=a[0], z_tg=a[1], actions=a[4], returns=a[5],
                       nonterminals=a[6], weights=a[7], kappa=a[8], gamma_n=a[9])
            assert a[0].shape[0] == B and a[1].shape[0] == 2 * B
        else:
            inp = dict(entry="plain", B=B, A=A, Z=N, q_on_s=a[0], q_tg_s=a[1], q_tg_ns=a[2], actions=a[3], returns=a[4],
                       nonterminals=a[5], weights=a[6], kappa=a[7], gamma_n=a[8])
        inp.update(alpha=alpha, tau=tau, clip=clip)
        T_ref, T_sc, b_ref, b_sc, _ = MR.targets(inp)
        R.assert_within(f"b of update {u}", seen["b"], b_ref, b_sc, Q.TAU)
        R.assert_within(f"T of update {u}", seen["T"], T_ref, T_sc, Q.TAU)
        (l_ref, l_sc), (g_ref, g_sc) = MR.loss_grad(inp, seen["T"])
        R.assert_within(f"loss of update {u}", seen["loss"], l_ref, l_sc, Q.TAU)
        d_ref, d_sc = MR.dz(inp, g_ref, g_sc) if fused else MR.grad_rows(inp, g_ref, g_sc)
        R.assert_within(f"grad of update {u}", seen["grad"], d_ref, d_sc, Q.TAU)
        assert torch.equal(seen["loss"], ag.last_loss)
        assert torch.equal(seen["T"], ag._stats["last"]["m"])
        ws = mem._last
        tidx, got = cpu(ws.tree_idx), cpu(ag.last_loss)
        last = np.array([i for i in range(len(tidx)) if tidx[i] not in tidx[i + 1:]])
        assert_bits_equal(cpu(mem.transitions.tree)[tidx[last]], np.sqrt(got)[last], f"priorities of update {u}")
        if u == 0 and not ag.augment_shift and not ag.augment_intensity:
            with torch.no_grad():   # the rows the kernel read are the nets' forwards of the batch's states
                tg = ag.target_net
                want = tg.head().forward(tg.features_nograd(torch.cat([ws.states, ws.next_states])))[0] if fused else \
                    tg.logits(torch.cat([ws.states, ws.next_states]))
            torch.cuda.synchronize()
            got_t = a[1] if fused else torch.cat([a[1], a[2]])
            assert torch.allclose(got_t, want, rtol=1e-5, atol=1e-5), "the target rows are the target net's [s; s']"
            opt, on = ag.optimiser, ag.online_net
            p_after = opt.flat_param.clone()
            opt.flat_param.copy_(p_before)     # the online rows: its forward of s with the parameters it updated from
            with torch.no_grad():
                want = on.head().forward(on.features_nograd(ws.states))[0] if fused else on.logits(ws.states)
            opt.flat_param.copy_(p_after)
            torch.cuda.synchronize()
            assert a[0].shape == want.shape
            assert torch.allclose(a[0], want, rtol=1e-5, atol=1e-5), "the online rows are the online net's s"


# ---- whole updates against float64 -----------------------------------------------------------------------------------------
MUNCH_CASES = [
    _row("quantile", "none", "fixed", "adam", "hard", "off", "off", "off", 32, "fused", "c-h512", "pending"),
    _row("quantile", "shift", "fixed", "adam", "polyak", "off", "off", "on", 64, "fused", "c-h64", "flushed"),
    _row("quantile", "none", "annealed", "adamw", "hard", "off", "on", "off", 32, "fused", "de-h256", "pending"),
    _row("quantile", "none", "fixed", "adam", "hard", "off", "off", "on", 32, "library", "c-h64", "flushed"),
    _row("quantile", "intensity", "annealed", "adamw", "polyak", "on", "on", "on", 32, "fused", "de-h256", "pending"),
]


_H_BEFORE_REDO = {}


def _sides_s(ag, ws, p_before):
    """The ReLU sides of the learner's own fp32 forward of the online rows of s (the only online rows under Munchausen),
    with the parameters it updated from: the conv layers recomputed (the same cuDNN calls on the same rows), the hidden
    layer from the fused head's h buffer of the update's B rows, or the library's NoisyLinear layers.  A ReDo pass after
    the update scores the same B rows through the same head buffers, so where one ran in this learn() the buffer is
    taken as it stood before it."""
    on, opt = ag.online_net, ag.optimiser
    H, B = on.hidden_size, ws.B
    fused = ag._fused_path(B)
    if fused:
        snap = _H_BEFORE_REDO.get(id(ag))
        h = snap[1] if snap is not None and snap[0] == ag._learn_calls else on.head()._scratch[B]["h"].clone()
    p_after = opt.flat_param.clone()
    opt.flat_param.copy_(p_before)
    with torch.no_grad():
        if fused:
            acts = on.conv_forward_saving(ws.states)[1:]
        else:
            acts, x = [], ws.states
            for m in on.convs:
                x = m(x)
                if isinstance(m, torch.nn.ReLU):
                    acts.append(x)
            x = on.features(ws.states)
            h = torch.cat([on.fc_h_v(x), on.fc_h_a(x)], 1)
    opt.flat_param.copy_(p_after)
    return [(a > 0).double() for a in acts], [(h[:, :H] > 0).double(), (h[:, H:] > 0).double()]


@pytest.mark.parametrize("c", MUNCH_CASES, ids=[case_id(c) for c in MUNCH_CASES])
def test_update_trajectory_against_float64(c, tmp_path, monkeypatch):
    """test_gpu_update_f64's trajectory check as it stands -- gather, loss, priorities, per-element gradients, optimiser,
    target, resets, ReDo and statistics, update by update -- with args.munchausen set, the Munchausen loss kernel as the
    loss node, and tests/munchausen_update_ref.py as the float64 reference: the online net on s, pi and l from the
    learner's own fp32 target rows of [s; s'] (the target head's output buffer), the s' quantiles in float64."""
    import munchausen_update_ref as MU
    import test_gpu_update_f64 as TU
    kwargs, kernels = TU.agent_kwargs, TU._expected_kernels

    def agent_kwargs(case):
        return dict(kwargs(case), munchausen=True)

    def expected(case, ag):
        gather, loss, bwd = kernels(case, ag)
        return gather, {"k_qr_dueling": "k_qr_dueling_munchausen", "k_qr": "k_qr_munchausen"}[loss], bwd

    def own_target_rows(ag, ws):
        return ag.target_net.head()._scratch[2 * ws.B]["z"].clone()

    def reference(*a, **k):
        alpha, tau, clip = agent_of[0].munchausen
        return MU.update_ref(*a, **k, alpha=alpha, tau=tau, clip=clip)

    agent_of = []
    from rainbow_b200.agent import Agent
    orig_init, orig_redo = Agent.__init__, Agent.recycle_dormant

    def redo(self, *a, **k):
        buf = self.online_net.head()._scratch.get(self.batch_size)
        if buf is not None:
            _H_BEFORE_REDO[id(self)] = (self._learn_calls, buf["h"].clone())
        return orig_redo(self, *a, **k)
    monkeypatch.setattr(Agent, "recycle_dormant", redo)

    def init(self, *a, **k):
        orig_init(self, *a, **k)
        agent_of.append(self)
    monkeypatch.setattr(Agent, "__init__", init)
    monkeypatch.setattr(TU, "agent_kwargs", agent_kwargs)
    monkeypatch.setattr(TU, "_expected_kernels", expected)
    monkeypatch.setattr(TU, "_sides", _sides_s)
    monkeypatch.setattr(TU, "_own_ns_rows", own_target_rows)
    monkeypatch.setattr(TU.U, "update_ref", reference)
    TU.test_update_trajectory_against_float64(c, tmp_path, monkeypatch)
    assert len(agent_of) == 1 and agent_of[0].munchausen is not None
