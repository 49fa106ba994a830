"""HL-Gauss targets on the H100: rb_c51_hlg_loss_grad and rb_c51_dueling_hlg_loss_grad per element against
tests/hlg_ref.py over the grid (Z 2 / 51 / 101, A 1 / 6 / 18, B 1 / 32 / 512, sigma / dz 0.1 / 0.75 / 4, supports pm10 /
0to20 / pm100), with guard rows, graph replay, the optional outputs and refused calls; y bitwise against the stated fp32
order; and the learner: the update graph, graph replay against eager with every composable switch on, resume, the
checkpoint's refusals, the annealed horizon, acting, the statistics and test_gpu_update_f64's whole-update trajectories."""
import html
import json
import re
import types

import numpy as np
import pytest
import torch

import c51_ref as C
import head_ref as R
import hlg_ref as H
from helpers import assert_bits_equal
from test_gpu_augment import update_graph
from test_gpu_head_f64 import graph_kernels
from test_gpu_parity import DEV, FakeEnv, cpu, make_args, synthetic_ring
from update_cases import _row, case_id

pytestmark = pytest.mark.gpu

NAN = float("nan")
GUARD = 3
CAP = 8192
HLG = dict(categorical_target="hl_gauss")


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


def run(entry, inp, sigma=None, optional=True, check=True):
    """One launch of an HL-Gauss entry into prefilled outputs with GUARD rows past each: (loss, dz or grad, m, a*, y);
    optional=False passes null m_out / astar_out / y_out (those three come back untouched); check=False expects the call
    to be refused with RB_ERR_INVAL."""
    B, A, Z = inp["B"], inp["A"], inp["Z"]
    sigma = inp["sigma"] if sigma is None else sigma
    loss, aout, m, y = _nan(B + GUARD), _nan(B + GUARD, dtype=torch.int64), _nan(B + GUARD, Z), _nan(B + GUARD)
    opt = (m.data_ptr(), aout.data_ptr(), y.data_ptr()) if optional else (None, None, None)
    common = (inp["actions"].data_ptr(), inp["returns"].data_ptr(), inp["nonterminals"].data_ptr(),
              inp["weights"].data_ptr(), inp["support"].data_ptr(), C.f32(inp["vmin"]), C.f32(inp["vmax"]),
              C.f32(inp["dz"]), C.f32(inp["gamma_n"]), sigma)
    if entry == "plain":
        g = _nan(B + GUARD, A, Z)
        rc = lib().rb_c51_hlg_loss_grad(inp["q_on_s"].data_ptr(), inp["q_on_ns"].data_ptr(), inp["q_tg_ns"].data_ptr(),
                                        *common, B, A, Z, loss.data_ptr(), g.data_ptr(), *opt, stream())
    else:
        g = _nan(B + GUARD, Z + A * Z)
        rc = lib().rb_c51_dueling_hlg_loss_grad(inp["z_on"].data_ptr(), inp["z_tg"].data_ptr(), A, Z, *common, B,
                                                loss.data_ptr(), g.data_ptr(), *opt, stream())
    assert rc == (0 if check else -22), lib().rb_last_error()
    return loss, g, m, aout, y


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


def target_values(inp, astar):
    """ybar per row, bitwise as the loss kernels form it: rb_q_values on the target rows (the dueling combination and
    c51_expected_value the loss kernels share) at a*."""
    B, A, Z = inp["B"], inp["A"], inp["Z"]
    if inp["entry"] == "plain":    # a dueling row with zero value and advantage q reproduces q only up to the mean: use
        return None                # the dueling entry for the bitwise check
    q = _nan(B, A)
    a, v = _nan(B, dtype=torch.int64), _nan(B)
    assert lib().rb_q_values(inp["z_tg"].data_ptr(), B, A, Z, inp["support"].data_ptr(), q.data_ptr(), a.data_ptr(),
                             v.data_ptr(), stream()) == 0
    return q[torch.arange(B, device=DEV), astar.long()]


# (entry, B, A, Z, support, ratio): every entry meets Z 2 / 51 / 101, A 1 / 6 / 18, B 1 / 32 / 512, all three ratios and
# all three supports
_ZA = [(Z, A) for Z in (2, 51, 101) for A in (1, 6, 18)]
GRID = [(e, (32, 512, 1)[(i + k) % 3], A, Z, ("pm10", "0to20", "pm100")[(i + 2 * k) % 3], H.RATIOS[(2 * i + k) % 3])
        for e in ("plain", "dueling") for i, (Z, A) in enumerate(_ZA) for k in (0, 1)]


@pytest.mark.parametrize("case", GRID, ids=[f"{c[0]}-B{c[1]}-A{c[2]}-Z{c[3]}-{c[4]}-s{c[5]:g}" for c in GRID])
def test_entries_against_float64(case, tmp_path):
    entry, B, A, Z, sup, ratio = case
    inp = C.to(H.make_inputs(entry, B, A, Z, sup, 5 + B + A + Z, ratio), DEV)
    eager = run(entry, inp)
    _, outs, dot = graph_kernels(lambda: run(entry, inp), tmp_path / "h.dot")
    kname = "k_c51_dueling_hlg" if entry == "dueling" else "k_c51_hlg"
    r = 2 if Z <= 64 else 4
    assert re.search(r"{}(ILi{}EE|<\s*{}\s*>)".format(kname, r, r), dot), f"{kname}<{r}> ran"
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
    ev, evs = C.expected_values(ci)
    ok = C.astar_ok(ev, evs, astar.cpu())
    assert bool(ok.all()), f"a* outside the bound on {int((~ok).sum())} rows"
    assert bool(C.first_of_identical(ci, astar.cpu()).all()), "a tie goes to the first action"
    (y_ref, ey), (m_ref, em) = H.target(ci, astar.cpu())
    R.assert_within("y", y.cpu(), y_ref, ey, 1.0)
    R.assert_within("m", m.cpu(), m_ref, em, 1.0)
    assert bool((m >= 0).all()) and bool(((m.double().sum(1) - 1).abs() <= 1e-5).all())
    (l_ref, l_sc), (g_ref, g_sc) = C.loss_grad(ci, m.cpu())
    R.assert_within("loss", loss.cpu(), l_ref, l_sc, C.TAU)
    d_ref, d_sc = C.dueling_dz(ci, g_ref, g_sc) if entry == "dueling" else _grad_rows(ci, g_ref, g_sc)
    R.assert_within("grad", g.cpu(), d_ref.reshape(g.shape), d_sc.reshape(g.shape), C.TAU)
    assert bool((g[inp["weights"] == 0] == 0).all()), "rows of weight 0 have an exactly zero gradient"
    lo, hi = C.f32(inp["vmin"]), C.f32(inp["vmax"])
    assert bool(((y >= lo) & (y <= hi)).all()), "y is clamped to the support"
    # y bitwise in the stated order, from ybar as the loss kernels form it
    yb = target_values(inp, astar)
    if yb is not None:
        f = np.float32
        sc = (cpu(inp["nonterminals"]).reshape(-1).astype(f) * f(inp["gamma_n"])).astype(f)
        want = np.clip((cpu(inp["returns"]).astype(f) + (sc * cpu(yb)).astype(f)).astype(f), f(lo), f(hi))
        assert_bits_equal(cpu(y), want, "y against fl32(r + fl32(sc ybar)), clamped")


def test_refused_calls_write_nothing():
    for entry in ("plain", "dueling"):
        inp = C.to(H.make_inputs(entry, 8, 6, 51, "pm10", 3, 0.75), DEV)
        for bad in (NAN, 0.0, -1.0, float("inf"), 1e-40):
            outs = run(entry, inp, sigma=bad, check=False)
            assert lib().rb_last_error().decode().startswith("rb_c51"), bad
            torch.cuda.synchronize()
            for t in outs:
                assert bool((t == -7).all()) if t.dtype == torch.int64 else bool(torch.isnan(t).all()), bad


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
    names, dots = {}, {}
    for tag, extra in (("c51", dict()), ("off", dict(categorical_target="projection")), ("hlg", HLG)):
        names[tag] = update_graph(_agent(**kw, **extra), _memory(), tmp_path / f"{tag}.dot", monkeypatch)
        dots[tag] = html.unescape(open(tmp_path / f"{tag}.dot").read())
    assert names["off"] == names["c51"], "categorical_target 'projection' leaves the update graph as it is"
    parent = "k_c51" if head == "library" else "k_c51_dueling"
    own = lambda ks: [k for k in ks if k.startswith("k_")]
    assert own(names["hlg"]) == [{parent: parent + "_hlg"}.get(k, k) for k in own(names["c51"])]
    assert own(names["hlg"]).count(parent + "_hlg") == 1 and parent not in own(names["hlg"])
    assert len(names["hlg"]) == len(names["c51"]), "the same node count"


@pytest.mark.parametrize("head", ["fused", "library", "truncation"])
def test_graph_replay_equals_eager(head):
    kw = dict(ALL, **HLG)
    mem_kw = dict(MEM_ALL)
    if head == "library":
        kw["fused_head"] = False
    if head == "truncation":
        kw, mem_kw = dict(HLG, augment_shift=4, target_tau=0.005, learn_stats=8, bootstrap_truncation=True), \
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
    kw = dict(augment_shift=4, hl_gauss_sigma=1.5, **HLG)
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
    assert (hp["categorical_target"], hp["hl_gauss_sigma"]) == ("hl_gauss", 1.5)
    ag, mem = ck_agent(seed=77, **kw), _fresh_memory()
    ag.load_checkpoint(str(tmp_path / "ck"), mem)
    for step in range(save_at, total):
        if step > save_at:
            _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _assert_same(run_a, _state(ag, mem, losses))

    plain = ck_agent(augment_shift=4)
    plain.save_checkpoint(str(tmp_path / "plain"))
    hp = json.load(open(tmp_path / "plain" / "rank0" / "manifest.json"))["hyper_parameters"]
    assert "categorical_target" not in hp and "hl_gauss_sigma" not in hp
    ag.save_checkpoint(str(tmp_path / "h"))
    _refused(ck_agent(seed=8, **kw), None, str(tmp_path / "plain"), match="categorical target")
    _refused(plain, None, str(tmp_path / "h"), match="categorical target")
    _refused(ck_agent(seed=8, **dict(kw, hl_gauss_sigma=0.75)), None, str(tmp_path / "h"), match="categorical target")


@pytest.mark.parametrize("case", ["fused-pending", "batch64", "c3", "library-head"])
def test_annealed_horizon_is_the_fixed_horizon(case, monkeypatch):
    """test_gpu_horizon's check as it stands, with both agents built with HL-Gauss targets."""
    import test_gpu_horizon as TH
    orig = TH._agent
    monkeypatch.setattr(TH, "_agent", lambda seed=5, **kw: orig(seed, **dict(kw, **HLG)))
    TH.test_annealed_update_is_the_plain_update_at_its_horizon(case)


def test_acting_and_evaluation_are_unchanged():
    kw = dict(architecture="data-efficient", hidden_size=64)
    h, plain = _agent(**kw, **HLG), _agent(**kw)
    val, _ = synthetic_ring(256, seed=4)
    states = val.iter_states(0, 8)
    for i in range(4):
        assert h.act(states[i]) == plain.act(states[i])
        assert h.evaluate_q(states[i]) == plain.evaluate_q(states[i])
    assert torch.equal(h.evaluate_q_batch(states), plain.evaluate_q_batch(states))
    assert h.evaluate_q_memory(val) == plain.evaluate_q_memory(val)


def test_learn_stats_hold_the_histogram_mean():
    ag = _agent(learn_stats=8, **HLG)
    mem = _memory()
    for _ in range(3):
        ag.reset_noise()
        ag.learn(mem)
    torch.cuda.synchronize()
    rec = ag.learn_stats()
    loss = cpu(ag.last_loss).astype(np.float64)
    assert rec["loss_mean"][-1] == pytest.approx(float(loss.mean()), rel=1e-6)
    m = cpu(ag._stats["last"]["m"]).astype(np.float64)
    assert np.isfinite(m).all() and np.allclose(m.sum(1), 1.0, atol=1e-5)
    tv = m @ cpu(ag.support).astype(np.float64)
    assert rec["target_mean"][-1] == pytest.approx(float(tv.mean()), rel=1e-5, abs=1e-5), "target_mean = sum_k m_k z_k"


# ---- whole updates against float64 -----------------------------------------------------------------------------------------
HLG_CASES = [
    _row("categorical", "none", "fixed", "adam", "hard", "off", "off", "off", 32, "fused", "c-h512", "pending"),
    _row("categorical", "shift", "fixed", "adam", "polyak", "off", "off", "on", 64, "fused", "c-h512", "flushed"),
    _row("categorical", "none", "annealed", "adamw", "hard", "off", "on", "off", 32, "fused", "c-h512", "pending"),
    _row("categorical", "none", "fixed", "adam", "hard", "off", "off", "on", 32, "library", "c-h64", "flushed"),
]


@pytest.mark.parametrize("c", HLG_CASES, ids=[case_id(c) for c in HLG_CASES])
def test_update_trajectory_against_float64(c, tmp_path, monkeypatch):
    """test_gpu_update_f64's trajectory check as it stands, with args.categorical_target = "hl_gauss", the HL-Gauss kernel
    as the loss node, and tests/hlg_ref.py's histogram in place of the projection in the float64 update (the float64
    target rows give ybar; the bound is hlg_ref's for y and m)."""
    import test_gpu_update_f64 as TU
    import update_ref as U
    kwargs, kernels = TU.agent_kwargs, TU._expected_kernels
    agent_of = []

    def agent_kwargs(case):
        return dict(kwargs(case), **HLG)

    def expected(case, ag):
        gather, loss, bwd = kernels(case, ag)
        return gather, loss + "_hlg", bwd

    def projection(inp, astar):
        ag = agent_of[0]
        inp = dict(_cpu_inp(inp), sigma=H.sigma_of(ag.hl_gauss_sigma, ag.delta_z))
        _, (m, em) = H.target(inp, astar.cpu())
        return m.to(astar.device), (em / C.TAU).to(astar.device)

    from rainbow_b200.agent import Agent
    orig_init = Agent.__init__

    def init(self, *a, **k):
        orig_init(self, *a, **k)
        agent_of.append(self)
    monkeypatch.setattr(Agent, "__init__", init)
    monkeypatch.setattr(U, "C", types.SimpleNamespace(**dict(vars(C), projection=projection)))
    monkeypatch.setattr(TU, "agent_kwargs", agent_kwargs)
    monkeypatch.setattr(TU, "_expected_kernels", expected)
    TU.test_update_trajectory_against_float64(c, tmp_path, monkeypatch)
