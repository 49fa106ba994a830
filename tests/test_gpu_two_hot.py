"""Two-hot targets on the H100: rb_c51_twohot_loss_grad, rb_c51_dueling_twohot_loss_grad and their _vt twins per element
against tests/twohot_ref.py over the grid (Z 2 / 51 / 101, A 1 / 6 / 18, B 1 / 32 / 512, supports pm10 / 0to20 / pm100,
value rescaling off, eps 1e-3 and eps 0), with guard rows, graph replay, the optional outputs and refused calls; bitwise
against the projection entries on rows whose target distribution is a point mass; and the learner: the update graph, graph
replay against eager with every composable switch on, resume, the checkpoint's refusals, the annealed horizon, acting, the
statistics and test_gpu_update_f64's whole-update trajectories."""
import json
import re
import types

import numpy as np
import pytest
import torch

import c51_ref as C
import head_ref as R
import twohot_ref as T
from helpers import assert_bits_equal
from test_gpu_augment import update_graph
from test_gpu_head_f64 import graph_kernels
from test_gpu_parity import DEV, FakeEnv, cpu, make_args, synthetic_ring
from update_cases import _row, case_id

pytestmark = pytest.mark.gpu

NAN = float("nan")
GUARD = 3
CAP = 8192
TH = dict(categorical_target="two_hot")
VT = dict(value_transform="rescale")


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


def _nan(*shape, dtype=torch.float32):
    if dtype == torch.int64:
        return torch.full(shape, -7, dtype=dtype, device=DEV)
    return torch.full(shape, NAN, dtype=dtype, device=DEV)


def _common(inp):
    return (inp["actions"].data_ptr(), inp["returns"].data_ptr(), inp["nonterminals"].data_ptr(),
            inp["weights"].data_ptr(), inp["support"].data_ptr(), C.f32(inp["vmin"]), C.f32(inp["vmax"]),
            C.f32(inp["dz"]), C.f32(inp["gamma_n"]))


def run(entry, inp, optional=True, check=True, eps=None):
    """One launch of a two-hot entry (the _vt twin when inp holds eps) into prefilled outputs with GUARD rows past each:
    (loss, dz or grad, m, a*, y); optional=False passes null m_out / astar_out / y_out (those three come back untouched);
    check=False expects the call to be refused with RB_ERR_INVAL; eps overrides inp's."""
    B, A, Z = inp["B"], inp["A"], inp["Z"]
    vt = "eps" in inp
    loss, aout, m, y = _nan(B + GUARD), _nan(B + GUARD, dtype=torch.int64), _nan(B + GUARD, Z), _nan(B + GUARD)
    opt = (m.data_ptr(), aout.data_ptr(), y.data_ptr()) if optional else (None, None, None)
    tail = (inp["support_q"].data_ptr(), inp["eps"] if eps is None else eps) if vt else ()
    if entry == "plain":
        g = _nan(B + GUARD, A, Z)
        fn = lib().rb_c51_twohot_vt_loss_grad if vt else lib().rb_c51_twohot_loss_grad
        rc = fn(inp["q_on_s"].data_ptr(), inp["q_on_ns"].data_ptr(), inp["q_tg_ns"].data_ptr(), *_common(inp), B, A, Z,
                loss.data_ptr(), g.data_ptr(), *opt, *tail, stream())
    else:
        g = _nan(B + GUARD, Z + A * Z)
        fn = lib().rb_c51_dueling_twohot_vt_loss_grad if vt else lib().rb_c51_dueling_twohot_loss_grad
        rc = fn(inp["z_on"].data_ptr(), inp["z_tg"].data_ptr(), A, Z, *_common(inp), B, loss.data_ptr(), g.data_ptr(),
                *opt, *tail, stream())
    assert rc == (0 if check else -22), lib().rb_last_error()
    return loss, g, m, aout, y


def run_projection(entry, inp):
    """The projection entry (rb_c51(_dueling)(_vt)_loss_grad) on the same inputs: (loss, dz or grad, m, a*)."""
    B, A, Z = inp["B"], inp["A"], inp["Z"]
    vt = "eps" in inp
    loss, aout, m = _nan(B + GUARD), _nan(B + GUARD, dtype=torch.int64), _nan(B + GUARD, Z)
    tail = (inp["support_q"].data_ptr(), inp["eps"]) if vt else ()
    if entry == "plain":
        g = _nan(B + GUARD, A, Z)
        fn = lib().rb_c51_vt_loss_grad if vt else lib().rb_c51_loss_grad
        rc = fn(inp["q_on_s"].data_ptr(), inp["q_on_ns"].data_ptr(), inp["q_tg_ns"].data_ptr(), *_common(inp), B, A, Z,
                loss.data_ptr(), g.data_ptr(), m.data_ptr(), aout.data_ptr(), *tail, stream())
    else:
        g = _nan(B + GUARD, Z + A * Z)
        fn = lib().rb_c51_dueling_vt_loss_grad if vt else lib().rb_c51_dueling_loss_grad
        rc = fn(inp["z_on"].data_ptr(), inp["z_tg"].data_ptr(), A, Z, *_common(inp), B, loss.data_ptr(), g.data_ptr(),
                m.data_ptr(), aout.data_ptr(), *tail, stream())
    assert rc == 0, lib().rb_last_error()
    return loss, g, m, aout


def _guards(outs, B):
    for t in outs:
        bad = t[B:] != -7 if t.dtype == torch.int64 else ~torch.isnan(t[B:])
        assert not bool(bad.any()), "written past its last row"


def _grad_rows(inp, g, gs):
    B, A, Z = inp["B"], inp["A"], inp["Z"]
    full = torch.zeros(B, A, Z, dtype=torch.float64)
    fs = torch.zeros(B, A, Z, dtype=torch.float64)
    rows, acts = torch.arange(B), inp["actions"].long().cpu()
    full[rows, acts], fs[rows, acts] = g.cpu(), gs.cpu()
    return full, fs


def _cpu_inp(inp):
    return {k: (v.cpu() if isinstance(v, torch.Tensor) else v) for k, v in inp.items()}


def _inputs(entry, B, A, Z, sup, eps, seed):
    return C.to(T.make_inputs(entry, B, A, Z, sup, seed, eps), DEV)


# (entry, B, A, Z, support, eps): every entry meets Z 2 / 51 / 101, A 1 / 6 / 18, B 1 / 32 / 512, all three supports and
# value rescaling off, at eps 1e-3 and at eps 0
_ZA = [(Z, A) for Z in (2, 51, 101) for A in (1, 6, 18)]
_EPS = (None, 1e-3, 0.0)
GRID = [(e, (32, 512, 1)[(i + k) % 3], A, Z, ("pm10", "0to20", "pm100")[(i + 2 * k) % 3], _EPS[(2 * i + k) % 3])
        for e in ("plain", "dueling") for i, (Z, A) in enumerate(_ZA) for k in (0, 1, 2)]


@pytest.mark.parametrize("case", GRID, ids=[f"{c[0]}-B{c[1]}-A{c[2]}-Z{c[3]}-{c[4]}-{'off' if c[5] is None else c[5]}"
                                            for c in GRID])
def test_entries_against_float64(case, tmp_path):
    entry, B, A, Z, sup, eps = case
    inp = _inputs(entry, B, A, Z, sup, eps, 5 + B + A + Z)
    eager = run(entry, inp)
    _, outs, dot = graph_kernels(lambda: run(entry, inp), tmp_path / "t.dot")
    kname = "k_c51_dueling_twohot" if entry == "dueling" else "k_c51_twohot"
    r, v = (2 if Z <= 64 else 4), int(eps is not None)
    assert re.search(r"{}(ILi{}ELb{}EE|<\s*{}\s*,\s*{}\s*>)".format(kname, r, v, r, ("false", "true")[v]), dot), \
        f"{kname}<{r}, {bool(v)}> ran"
    _guards(outs, B)
    _guards(eager, B)
    for name, a, b in zip(("loss", "grad", "m", "a*", "y"), eager, outs):
        assert torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0)), f"{name}: eager launch and graph replay differ"
    bare = run(entry, inp, optional=False)
    for name, a, b in zip(("loss", "grad"), eager[:2], bare[:2]):
        assert torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0)), f"{name}: the call without the optional outputs differs"
    assert bool(torch.isnan(bare[2]).all() and (bare[3] == -7).all() and torch.isnan(bare[4]).all())
    loss, g, m, astar, y = (t[:B] for t in outs)
    torch.cuda.synchronize()
    ci = _cpu_inp(inp)
    ev, evs = T.expected_values(ci)
    ok = C.astar_ok(ev, evs, astar.cpu())
    assert bool(ok.all()), f"a* outside the bound on {int((~ok).sum())} rows"
    assert bool(C.first_of_identical(ci, astar.cpu()).all()), "a tie goes to the first action"
    (y_ref, ey), (m_ref, em) = T.target(ci, astar.cpu())
    R.assert_within("y", y.cpu(), y_ref, ey, 1.0)
    R.assert_within("m", m.cpu(), m_ref, em, 1.0)
    # m from the kernel's own y: at most two adjacent non-zeros, within the split's rounding of that y
    _, (m_own, em_own) = T.target(ci, astar.cpu(), y=y)
    R.assert_within("m (from y)", m.cpu(), m_own, em_own, 1.0)
    assert bool(((m != 0).sum(1) <= 2).all()) and bool((m >= 0).all())
    (l_ref, l_sc), (g_ref, g_sc) = C.loss_grad(ci, m.cpu())     # the loss row from the kernel's m, as c51_ref blames it
    R.assert_within("loss", loss.cpu(), l_ref, l_sc, C.TAU)
    d_ref, d_sc = C.dueling_dz(ci, g_ref, g_sc) if entry == "dueling" else _grad_rows(ci, g_ref, g_sc)
    R.assert_within("grad", g.cpu(), d_ref.reshape(g.shape), d_sc.reshape(g.shape), C.TAU)
    assert bool((g[inp["weights"] == 0] == 0).all()), "rows of weight 0 have an exactly zero gradient"
    lo, hi = C.f32(inp["vmin"]), C.f32(inp["vmax"])
    assert bool(((y >= lo) & (y <= hi)).all()), "y is clamped to the support"
    for i in range(B):   # the moved rows: clamped, and a y exactly on an atom is a one-hot
        if i % 11 == 9:
            assert float(y[i]) == lo and float(m[i, 0]) == 1.0, i
        if i % 11 == 10:
            assert float(y[i]) == hi, i
        if i % 11 == 6 and bool((inp["support"] == y[i]).any()):
            b = (np.float32(cpu(y[i:i + 1])[0]) - np.float32(lo)) / np.float32(inp["dz"])
            if float(b) == float(np.floor(b)):
                assert float(m[i].max()) == 1.0 and int((m[i] != 0).sum()) == 1, i


def _point_mass_inputs(entry, B, A, Z, sup, eps, seed):
    """Inputs whose target rows are point masses: every action's target(s') has one atom j_i at 0 and every other atom near
    -300 (the dueling layout: the one-hot in the value stream, advantages N(0, 0.01)), so every other atom's expf underflows
    to exactly 0 and the target's expected value is exactly s_j (s~_j)."""
    inp = T.make_inputs(entry, B, A, Z, sup, seed, eps)
    g = torch.Generator().manual_seed(seed + 31)
    j = torch.randint(0, Z, (B,), generator=g)
    if entry == "plain":
        q = -300.0 + 0.01 * torch.randn(B, A, Z, generator=g)
        q[torch.arange(B), :, j] = 0.0
        inp["q_tg_ns"] = q
    else:
        z = 0.01 * torch.randn(B, Z + A * Z, generator=g)
        z[:, :Z] = -300.0
        z[torch.arange(B), j] = 0.0
        inp["z_tg"] = z
    return C.to(inp, DEV)


@pytest.mark.parametrize("entry", ["plain", "dueling"])
@pytest.mark.parametrize("eps", [None, 1e-3, 0.0])
@pytest.mark.parametrize("B,A,Z,sup", [(32, 6, 51, "pm10"), (33, 18, 101, "0to20"), (7, 1, 2, "pm100")])
def test_point_mass_rows_are_the_projection_bitwise(entry, eps, B, A, Z, sup):
    """On rows whose target distribution at a* is a point mass on atom j, ybar is exactly s_j (s~_j under the transform),
    so y is the projection's one target atom and m, loss and dz / grad are the projection entry's, bitwise."""
    inp = _point_mass_inputs(entry, B, A, Z, sup, eps, 11 + Z)
    loss, g, m, astar, y = run(entry, inp)
    p_loss, p_g, p_m, p_astar = run_projection(entry, inp)
    torch.cuda.synchronize()
    assert_bits_equal(cpu(astar), cpu(p_astar), "a*")
    assert_bits_equal(cpu(m), cpu(p_m), "m")
    assert_bits_equal(cpu(loss), cpu(p_loss), "loss")
    assert_bits_equal(cpu(g), cpu(p_g), "dz" if entry == "dueling" else "grad")


def test_refused_calls_write_nothing():
    for entry in ("plain", "dueling"):
        inp = _inputs(entry, 8, 6, 51, "pm10", 1e-3, 3)
        for bad in (NAN, -1e-3, 1.5):
            outs = run(entry, inp, check=False, eps=bad)
            assert lib().rb_last_error().decode().startswith("rb_c51"), bad
            torch.cuda.synchronize()
            for t in outs:
                assert bool((t == -7).all()) if t.dtype == torch.int64 else bool(torch.isnan(t).all()), bad
        plain = _inputs(entry, 8, 6, 51, "pm10", None, 3)
        plain["B"] = 0
        outs = run(entry, plain, check=False)
        torch.cuda.synchronize()
        for t in outs:
            assert bool((t == -7).all()) if t.dtype == torch.int64 else bool(torch.isnan(t).all())


# ---- the learner -----------------------------------------------------------------------------------------------------------
ALL = dict(augment_shift=4, augment_intensity=0.05, target_tau=0.005, reset_interval=5, redo_interval=3,
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


@pytest.mark.parametrize("head", ["fused-b32", "fused-b64", "library"])
def test_update_graph_nodes(head, tmp_path, monkeypatch):
    kw = dict(batch_size=64) if head == "fused-b64" else (dict(fused_head=False) if head == "library" else dict())
    names = {}
    for tag, extra in (("c51", dict()), ("th", TH), ("vt", VT), ("th-vt", dict(TH, **VT))):
        names[tag] = update_graph(_agent(**kw, **extra), _memory(), tmp_path / f"{tag}.dot", monkeypatch)
    parent = "k_c51" if head == "library" else "k_c51_dueling"
    own = lambda ks: [k for k in ks if k.startswith("k_")]
    for base, twin in (("c51", "th"), ("vt", "th-vt")):
        assert own(names[twin]) == [{parent: parent + "_twohot"}.get(k, k) for k in own(names[base])]
        assert own(names[twin]).count(parent + "_twohot") == 1 and parent not in own(names[twin])
        assert len(names[twin]) == len(names[base]), "the same node count"


@pytest.mark.parametrize("head", ["fused", "library", "truncation", "rescale"])
def test_graph_replay_equals_eager(head):
    kw = dict(ALL, **TH)
    mem_kw = dict(MEM_ALL)
    if head == "library":
        kw["fused_head"] = False
    if head == "rescale":
        kw.update(VT)
    if head == "truncation":
        kw, mem_kw = dict(TH, augment_shift=4, target_tau=0.005, learn_stats=8, bootstrap_truncation=True), \
            dict(bootstrap_truncation=True)
    ga, ea = _agent(**kw), _agent(cuda_graph=False, **kw)
    gm, em = _memory(**mem_kw), _memory(**mem_kw)
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
    kw = dict(augment_shift=4, **TH)
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
    assert hp["categorical_target"] == "two_hot" and "hl_gauss_sigma" not in hp
    ag, mem = ck_agent(seed=77, **kw), _fresh_memory()
    ag.load_checkpoint(str(tmp_path / "ck"), mem)
    for step in range(save_at, total):
        if step > save_at:
            _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _assert_same(run_a, _state(ag, mem, losses))

    plain = ck_agent(augment_shift=4)
    plain.save_checkpoint(str(tmp_path / "plain"))
    hlg = ck_agent(augment_shift=4, categorical_target="hl_gauss")
    hlg.save_checkpoint(str(tmp_path / "hlg"))
    hp = json.load(open(tmp_path / "plain" / "rank0" / "manifest.json"))["hyper_parameters"]
    assert "categorical_target" not in hp
    ag.save_checkpoint(str(tmp_path / "th"))
    _refused(ck_agent(seed=8, **kw), None, str(tmp_path / "plain"), match="categorical target")
    _refused(plain, None, str(tmp_path / "th"), match="categorical target")
    _refused(ck_agent(seed=8, **kw), None, str(tmp_path / "hlg"), match="categorical target")
    _refused(hlg, None, str(tmp_path / "th"), match="categorical target")


@pytest.mark.parametrize("case", ["fused-pending", "batch64", "c3", "library-head"])
def test_annealed_horizon_is_the_fixed_horizon(case, monkeypatch):
    """test_gpu_horizon's check as it stands, with both agents built with two-hot targets."""
    import test_gpu_horizon as TGH
    orig = TGH._agent
    monkeypatch.setattr(TGH, "_agent", lambda seed=5, **kw: orig(seed, **dict(kw, **TH)))
    TGH.test_annealed_update_is_the_plain_update_at_its_horizon(case)


@pytest.mark.parametrize("vt", [False, True])
def test_acting_and_evaluation_are_unchanged(vt):
    kw = dict(architecture="data-efficient", hidden_size=64, **(VT if vt else {}))
    th, plain = _agent(**kw, **TH), _agent(**kw)
    val, _ = synthetic_ring(256, seed=4)
    states = val.iter_states(0, 8)
    for i in range(4):
        assert th.act(states[i]) == plain.act(states[i])
        assert th.evaluate_q(states[i]) == plain.evaluate_q(states[i])
    assert torch.equal(th.evaluate_q_batch(states), plain.evaluate_q_batch(states))
    assert th.evaluate_q_memory(val) == plain.evaluate_q_memory(val)


@pytest.mark.parametrize("vt", [False, True])
def test_learn_stats_hold_the_split_mean(vt):
    ag = _agent(learn_stats=8, **TH, **(VT if vt else {}))
    mem = _memory()
    for _ in range(3):
        ag.reset_noise()
        ag.learn(mem)
    torch.cuda.synchronize()
    rec = ag.learn_stats()
    loss = cpu(ag.last_loss).astype(np.float64)
    assert rec["loss_mean"][-1] == pytest.approx(float(loss.mean()), rel=1e-6)
    m = cpu(ag._stats["last"]["m"]).astype(np.float64)
    assert np.isfinite(m).all() and ((m != 0).sum(1) <= 2).all()
    tv = m @ cpu(ag.q_support if vt else ag.support).astype(np.float64)
    assert rec["target_mean"][-1] == pytest.approx(float(tv.mean()), rel=1e-5, abs=1e-5), "target_mean = sum_k m_k z_k"


# ---- whole updates against float64 -----------------------------------------------------------------------------------------
TH_CASES = [
    (_row("categorical", "none", "fixed", "adam", "hard", "off", "off", "off", 32, "fused", "c-h512", "pending"), False),
    (_row("categorical", "shift", "fixed", "adam", "polyak", "off", "off", "on", 64, "fused", "c-h512", "flushed"), False),
    (_row("categorical", "none", "annealed", "adamw", "hard", "off", "on", "off", 32, "fused", "c-h512", "pending"), False),
    (_row("categorical", "none", "fixed", "adam", "hard", "off", "off", "on", 32, "library", "c-h64", "flushed"), False),
    (_row("categorical", "none", "fixed", "adam", "hard", "off", "off", "off", 32, "fused", "c-h512", "pending"), True),
]


@pytest.mark.parametrize("c,vt", TH_CASES, ids=[case_id(c) + ("-rescale" if vt else "") for c, vt in TH_CASES])
def test_update_trajectory_against_float64(c, vt, tmp_path, monkeypatch):
    """test_gpu_update_f64's trajectory check as it stands, with args.categorical_target = "two_hot" (and value
    rescaling where vt), the two-hot kernel as the loss node, and tests/twohot_ref.py's split in place of the projection in
    the float64 update (the float64 target rows give ybar; the bound is twohot_ref's for m).  Under value rescaling the
    float64 arg-max takes the agent's q_support."""
    import test_gpu_update_f64 as TU
    import update_ref as U
    kwargs, kernels = TU.agent_kwargs, TU._expected_kernels
    agent_of = []

    def agent_kwargs(case):
        return dict(kwargs(case), **TH, **(VT if vt else {}))

    def expected(case, ag):
        gather, loss, bwd = kernels(case, ag)
        return gather, loss + "_twohot", bwd

    def projection(inp, astar):
        ag = agent_of[0]
        inp = _cpu_inp(inp)
        if vt:
            inp.update(support_q=ag.q_support.cpu(), eps=ag.value_transform_eps)
        _, (m, em) = T.target(inp, astar.cpu())
        return m.to(astar.device), (em / C.TAU).to(astar.device)

    orig_choices = U.argmax_choices

    def choices(q, L, dist, support=None):
        return orig_choices(q, L, dist, agent_of[0].q_support.to(q.device).double() if vt else support)

    from rainbow_b200.agent import Agent
    orig_init = Agent.__init__

    def init(self, *a, **k):
        orig_init(self, *a, **k)
        agent_of.append(self)
    monkeypatch.setattr(Agent, "__init__", init)
    monkeypatch.setattr(U, "C", types.SimpleNamespace(**dict(vars(C), projection=projection)))
    monkeypatch.setattr(U, "argmax_choices", choices)
    monkeypatch.setattr(TU, "agent_kwargs", agent_kwargs)
    monkeypatch.setattr(TU, "_expected_kernels", expected)
    TU.test_update_trajectory_against_float64(c, tmp_path, monkeypatch)
