"""Risk-sensitive selection on the GPU: the six _risk entries (k_c51 / k_c51_dueling / k_qr / k_qr_dueling / k_q_select /
k_qr_select) and the learner under args.risk_measure (DESIGN.md §18).

* The kernels (the RISK instantiations: R | RISK_INST of the four loss kernels, RISK = true of the two select kernels),
  per element against tests/risk_ref.py over Z = N 51 / 128 (R = 2 / 4), A 1 / 3 / 6 / 18, B 1 / 32 / 512,
  CVaR eta 0.1 / 0.25 / 1 and Wang eta -0.75 / 0 / 0.75, with c51_ref's / qr_ref's row kinds (terminals, weight 0, sharp,
  constant and tied rows): a* within the bound of the reference's best (bit-identical rows: the first), and everything
  downstream held to c51_ref / qr_ref at the kernel's a*; on every row whose a* is the parent entry's, loss, dz / grad and
  m / theta equal the parent's bitwise; rows past B stay untouched; an eager launch equals a graph replay.  A constructed
  case where the mean and CVaR disagree by a wide margin.  CVaR values are the stated fp32 order bitwise.
* The learner: the update graph's nodes, graph replay against eager updates with every composable switch on, resume,
  checkpoint refusals in both directions, the annealed horizon, acting / evaluation on the learner's own head rows, and
  tests/test_gpu_update_f64.py's whole-update trajectories with a* from the risk reference."""
import html
import json
import re

import numpy as np
import pytest
import torch

import c51_ref as C
import head_ref as R
import qr_ref as Q
import risk_ref as RR
from helpers import assert_bits_equal
from test_gpu_augment import update_graph
from test_gpu_head_f64 import graph_kernels
from test_gpu_parity import DEV, FakeEnv, cpu, make_args, synthetic_ring
from update_cases import _row, case_id

pytestmark = pytest.mark.gpu

NAN = float("nan")
GUARD = 3
CAP = 8192
MEASURES = [("cvar", 0.1), ("cvar", 0.25), ("cvar", 1.0), ("wang", -0.75), ("wang", 0.0), ("wang", 0.75)]


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


def run(entry, inp, risk):
    """One launch of a loss entry (risk (kind, eta), or None: the parent) into prefilled outputs with GUARD rows past
    each: (loss, dz or grad, m or theta, a*)."""
    B, A, Z = inp["B"], inp["A"], inp["Z"]
    cat = entry.startswith("c51")
    loss, aout = _nan(B + GUARD), _nan(B + GUARD, dtype=torch.int64)
    mt = _nan(B + GUARD, Z)
    common = (inp["actions"].data_ptr(), inp["returns"].data_ptr(), inp["nonterminals"].data_ptr(),
              inp["weights"].data_ptr())
    tail = (() if risk is None else (RR.KINDS[risk[0]], risk[1])) + (stream(),)
    name = {"c51": "rb_c51{}_loss_grad", "c51_dueling": "rb_c51_dueling{}_loss_grad", "qr": "rb_qr{}_loss_grad",
            "qr_dueling": "rb_qr_dueling{}_loss_grad"}[entry].format("" if risk is None else "_risk")
    fn = getattr(lib(), name)
    c51 = (inp["support"].data_ptr(), C.f32(inp["vmin"]), C.f32(inp["vmax"]), C.f32(inp["dz"]), C.f32(inp["gamma_n"])) \
        if cat else (C.f32(inp["kappa"]), C.f32(inp["gamma_n"]))
    if entry in ("c51", "qr"):
        g = _nan(B + GUARD, A, Z)
        rc = fn(inp["q_on_s"].data_ptr(), inp["q_on_ns"].data_ptr(), inp["q_tg_ns"].data_ptr(), *common, *c51, B, A, Z,
                loss.data_ptr(), g.data_ptr(), mt.data_ptr(), aout.data_ptr(), *tail)
    else:
        g = _nan(B + GUARD, Z + A * Z)
        rc = fn(inp["z_on"].data_ptr(), inp["z_tg"].data_ptr(), A, Z, *common, *c51, B, loss.data_ptr(), g.data_ptr(),
                mt.data_ptr(), aout.data_ptr(), *tail)
    assert rc == 0, lib().rb_last_error()
    return loss, g, mt, aout


def select(z, A, Z, risk, support=None):
    """rb_q_values(_risk) / rb_qr_q_values(_risk) into prefilled outputs: (q [M][A], a [M], v [M])."""
    M = z.shape[0]
    q, a, v = _nan(M + GUARD, A), _nan(M + GUARD, dtype=torch.int64), _nan(M + GUARD)
    outs = (q.data_ptr(), a.data_ptr(), v.data_ptr())
    tail = (() if risk is None else (RR.KINDS[risk[0]], risk[1])) + (stream(),)
    if support is None:
        fn = lib().rb_qr_q_values if risk is None else lib().rb_qr_q_values_risk
        rc = fn(z.data_ptr(), M, A, Z, *outs, *tail)
    else:
        fn = lib().rb_q_values if risk is None else lib().rb_q_values_risk
        rc = fn(z.data_ptr(), M, A, Z, support.data_ptr(), *outs, *tail)
    assert rc == 0, lib().rb_last_error()
    return q, a, v


def _guards(outs, B):
    for t in outs:
        bad = t[B:] != -7 if t.dtype == torch.int64 else ~torch.isnan(t[B:])
        assert not bool(bad.any()), "written past its last row"


def make(entry, B, A, Z, seed):
    if entry.startswith("c51"):
        return C.to(C.make_inputs("plain" if entry == "c51" else "dueling", B, A, Z, "pm10", seed), DEV)
    return C.to(Q.make_inputs("plain" if entry == "qr" else "dueling", B, A, Z, 1.0, seed), DEV)


def _grad_rows(inp, g, gs):
    B, A, Z = inp["B"], inp["A"], inp["Z"]
    full, fs = torch.zeros(B, A, Z, dtype=torch.float64, device=g.device), torch.zeros(B, A, Z, dtype=torch.float64,
                                                                                       device=g.device)
    rows, acts = torch.arange(B, device=g.device), inp["actions"].long()
    full[rows, acts], fs[rows, acts] = g, gs
    return full, fs


# (entry, B, A, Z, measure, eta): every entry meets Z 51 / 128, A 1 / 3 / 6 / 18, B 1 / 32 / 512 and all six measures
_BS = (32, 512, 1)
GRID = [(e, _BS[(i + k) % 3], A, Z, *MEASURES[(2 * i + k + 3 * (Z == 128)) % 6])
        for e in ("c51", "c51_dueling", "qr", "qr_dueling")
        for i, (Z, A) in enumerate([(Z, A) for Z in (51, 128) for A in (1, 3, 6, 18)])
        for k in (0, 1)]


@pytest.mark.parametrize("case", GRID, ids=[f"{c[0]}-B{c[1]}-A{c[2]}-Z{c[3]}-{c[4]}{c[5]:g}" for c in GRID])
def test_loss_entries_against_float64(case, tmp_path):
    entry, B, A, Z, measure, eta = case
    risk = (measure, eta)
    inp = make(entry, B, A, Z, 11 + B + A + Z)
    eager = run(entry, inp, risk)
    _, outs, dot = graph_kernels(lambda: run(entry, inp, risk), tmp_path / "r.dot")
    assert re.search(r"k_{}(ILi(18|20)ELb0EE|<\s*(18|20)\s*,\s*false\s*>)".format(entry), dot), \
        "the RISK instantiation (R | RISK_INST, RISK_INST = 16) ran"
    _guards(outs, B)
    _guards(eager, B)
    for name, a, b in zip(("loss", "grad", "m", "a*"), eager, outs):
        assert torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0)), f"{name}: eager launch and graph replay differ"
    loss, g, mt, astar = (t[:B] for t in outs)
    Qv, err = RR.values(inp, "ns", measure, eta)
    ok = RR.astar_ok(Qv, err, astar)
    assert bool(ok.all()), f"a* outside the bound on {int((~ok).sum())} rows"
    assert bool(C.first_of_identical(inp, astar).all()), "a tie goes to the first action"
    if entry.startswith("c51"):
        m_ref, m_sc = C.projection(inp, astar)
        R.assert_within("m", mt, m_ref, m_sc, C.TAU)
        (l_ref, l_sc), (g_ref, g_sc) = C.loss_grad(inp, mt)
        tau = C.TAU
    else:
        T_ref, T_sc = Q.targets(inp, astar)
        R.assert_within("T", mt, T_ref, T_sc, Q.TAU)
        (l_ref, l_sc), (g_ref, g_sc) = Q.loss_grad(inp, mt)
        tau = Q.TAU
    R.assert_within("loss", loss, l_ref, l_sc, tau)
    d_ref, d_sc = C.dueling_dz(inp, g_ref, g_sc) if entry.endswith("dueling") else _grad_rows(inp, g_ref, g_sc)
    R.assert_within("grad", g, d_ref, d_sc, tau)
    assert bool((g[inp["weights"] == 0] == 0).all()), "rows of weight 0 have an exactly zero gradient"

    # bitwise the parent wherever the two arg-maxes agree
    p_loss, p_g, p_mt, p_astar = (t[:B] for t in run(entry, inp, None))
    same = astar == p_astar
    if measure == "cvar" and eta == 1.0 or measure == "wang" and eta == 0.0:
        assert float(same.float().mean()) > 0.5, "the neutral measures mostly pick the mean's a*"
    torch.cuda.synchronize()
    for name, a, b in (("loss", loss, p_loss), ("grad", g, p_g), ("m / theta", mt, p_mt)):
        assert_bits_equal(cpu(a[same]), cpu(b[same]), f"{name} where a* agrees")


def _disagreeing_quantiles(B, N):
    """Action 0: the higher mean (3.45) with a heavy lower tail (5 of 51 quantiles at -20); action 1: 1.5 everywhere."""
    n_tail = max(1, round(5 * N / 51))
    a0 = torch.cat([torch.full((n_tail,), -20.0), torch.full((N - n_tail,), 6.0)])
    return torch.stack([a0, torch.full((N,), 1.5)]).unsqueeze(0).expand(B, 2, N).contiguous()


@pytest.mark.parametrize("N", [51, 128])
def test_risk_and_mean_disagree(N):
    """CVaR 0.25 picks action 1 in every entry; the parents pick action 0, bitwise.  Through the dueling combination
    (value 0, the rows as advantages) the two actions become q_0 = (row_0 - 1.5) / 2 and q_1 = -q_0: action 0 keeps the
    higher mean (by 1.95) and the heavy lower tail, and CVaR prefers action 1 by more than 5."""
    B, A = 32, 2
    q = _disagreeing_quantiles(B, N)
    assert float(q[0, 0].mean() - q[0, 1].mean()) > 1.0
    risk = ("cvar", 0.25)
    base = Q.make_inputs("plain", B, A, N, 1.0, 3)
    plain = C.to(dict(base, q_on_ns=q, q_on_s=q, q_tg_ns=q), DEV)
    zrow = torch.cat([torch.zeros(B, N), q.reshape(B, A * N)], 1)
    duel = C.to(dict(Q.make_inputs("dueling", B, A, N, 1.0, 3), z_on=torch.cat([zrow, zrow]), z_tg=zrow), DEV)
    # categorical: 10% of the mass at V_min, 90% at 6 for action 0 (mean 4.4); all of it at 1.6 for action 1
    sup = torch.linspace(-10, 10, N)
    lp = torch.full((A, N), -1e4)
    lp[0, 0], lp[0, int(torch.argmin((sup - 6).abs()))] = float(np.log(0.1)), float(np.log(0.9))
    lp[1, int(torch.argmin((sup - 1.6).abs()))] = 0.0
    lg = lp.unsqueeze(0).expand(B, A, N).contiguous()
    cp = C.to(dict(C.make_inputs("plain", B, A, N, "pm10", 3), q_on_ns=lg, q_on_s=lg, q_tg_ns=lg), DEV)
    crow = torch.cat([torch.zeros(B, N), lg.reshape(B, A * N)], 1)
    cd = C.to(dict(C.make_inputs("dueling", B, A, N, "pm10", 3), z_on=torch.cat([crow, crow]), z_tg=crow), DEV)
    for entry, inp in (("qr", plain), ("qr_dueling", duel), ("c51", cp), ("c51_dueling", cd)):
        assert bool((run(entry, inp, risk)[3][:B] == 1).all()), entry
        assert bool((run(entry, inp, None)[3][:B] == 0).all()), f"{entry}: the parent takes the mean"
    zq, zc = zrow.to(DEV), crow.to(DEV)
    for z, s in ((zq, None), (zc, sup.to(DEV))):
        _, a, v = select(z, A, N, risk, s)
        _, pa, pv = select(z, A, N, None, s)
        assert bool((a[:B] == 1).all()) and bool((pa[:B] == 0).all())
        Qv, err = RR.select_values(z, A, N, *risk, support=s)
        R.assert_within("Q_beta", v[:B], Qv.max(1).values, err.max(1).values, 1.0)
        assert bool((Qv[:, 1] > Qv[:, 0] + 1.0).all()), "a wide margin"


# ---- the select entries ------------------------------------------------------------------------------------------------------
SELECT = [(dist, M, A, Z, *MEASURES[(i + 2 * j) % 6]) for dist in ("categorical", "quantile")
          for i, (M, A, Z) in enumerate([(1, 1, 51), (32, 3, 128), (512, 6, 51), (33, 18, 128), (5, 18, 51), (64, 6, 2)])
          for j in (0, 1)]


@pytest.mark.parametrize("case", SELECT, ids=[f"{c[0][:4]}-M{c[1]}-A{c[2]}-Z{c[3]}-{c[4]}{c[5]:g}" for c in SELECT])
def test_select_entries_against_float64(case, tmp_path):
    dist, M, A, Z, measure, eta = case
    g = torch.Generator().manual_seed(M + A + Z)
    z = (torch.randn(M, Z + A * Z, generator=g) * 2.0).to(DEV)
    z[::3] *= 15.0                                              # sharp rows
    sup = torch.linspace(-10, 10, Z, device=DEV) if dist == "categorical" else None
    risk = (measure, eta)
    eager = select(z, A, Z, risk, sup)
    _, outs, _ = graph_kernels(lambda: select(z, A, Z, risk, sup), tmp_path / "s.dot")
    _guards(outs, M)
    for a, b in zip(eager, outs):
        assert torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0)), "eager launch and graph replay differ"
    q, a, v = (t[:M] for t in outs)
    Qv, err = RR.select_values(z, A, Z, measure, eta, sup)
    R.assert_within("Q_beta", q, Qv, err, 1.0)
    assert bool(RR.astar_ok(Qv, err, a).all())
    assert torch.equal(v, q.gather(1, a.view(-1, 1)).view(-1)), "the value is the chosen action's"
    assert torch.equal(a, q.argmax(1)), "the first maximum wins"


@pytest.mark.parametrize("Z", [2, 51, 101, 128])
@pytest.mark.parametrize("eta", [0.1, 0.25, 1.0])
def test_cvar_values_are_the_stated_order_bitwise(Z, eta):
    """rb_q_values_risk / rb_qr_q_values_risk under CVaR equal the fp32 emulation of DESIGN.md §18's order bitwise, and
    the loss entries' a* is the first maximum of the same values."""
    M, A = 40, 6
    g = torch.Generator().manual_seed(Z)
    z = (torch.randn(M, Z + A * Z, generator=g) * 3.0).to(DEV)
    z[1::4] *= 10.0
    sup = torch.linspace(-10, 10, Z, device=DEV)
    x = RR.dueling32(z, A, Z)
    for s, emu in ((None, lambda: RR.emulate_quantile(x, "cvar", eta)),
                   (sup, lambda: RR.emulate_categorical(x, sup, "cvar", eta))):
        q, _, _ = select(z, A, Z, ("cvar", eta), s)
        want = emu()
        torch.cuda.synchronize()
        assert_bits_equal(cpu(q[:M]), cpu(want), "Q_beta")
    for entry in ("qr_dueling", "c51_dueling"):
        inp = make(entry, M, A, Z, 5)
        inp["z_on"][M:] = z
        astar = run(entry, inp, ("cvar", eta))[3][:M]
        xs = RR.dueling32(inp["z_on"][M:], A, Z)
        vals = RR.emulate_quantile(xs, "cvar", eta) if entry == "qr_dueling" else \
            RR.emulate_categorical(xs, inp["support"], "cvar", eta)
        assert torch.equal(astar, vals.argmax(1)), entry


@pytest.mark.parametrize("entry", ["c51", "c51_dueling", "qr", "qr_dueling"])
def test_refused_calls_write_nothing(entry):
    inp = make(entry, 8, 6, 51, 3)
    for kind, eta in (("cvar", 0.0), ("cvar", NAN), ("wang", float("inf"))):
        with pytest.raises(AssertionError):
            run(entry, inp, (kind, eta))
        torch.cuda.synchronize()
    # run() asserts on the return code before returning its outputs: check them by hand once
    B, A, Z = 8, 6, 51
    loss, aout = _nan(B), _nan(B, dtype=torch.int64)
    z = torch.zeros(B, Z + A * Z, device=DEV)
    q = _nan(B, A)
    rc = lib().rb_qr_q_values_risk(z.data_ptr(), B, A, Z, q.data_ptr(), aout.data_ptr(), loss.data_ptr(), 9, 0.5, stream())
    assert rc == -22
    torch.cuda.synchronize()
    assert bool(torch.isnan(q).all()) and bool((aout == -7).all()) and bool(torch.isnan(loss).all())


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


@pytest.mark.parametrize("dist", ["categorical", "quantile"])
def test_update_graph_nodes(dist, tmp_path, monkeypatch):
    names, dots = {}, {}
    for tag, kw in (("mean", dict()), ("off", dict(risk_measure="neutral")), ("risk", dict(risk_measure="wang"))):
        names[tag] = update_graph(_agent(distribution=dist, **kw), _memory(), tmp_path / f"{tag}.dot", monkeypatch)
        dots[tag] = html.unescape(open(tmp_path / f"{tag}.dot").read())
    assert names["off"] == names["mean"], "risk_measure 'neutral' leaves the update graph as it is"
    assert names["risk"] == names["mean"], "the same nodes, the risk instantiation in the parent's place"
    loss = "k_c51_dueling" if dist == "categorical" else "k_qr_dueling"
    flag = re.compile(loss + r"(ILi(18|20)ELb0EE|<\s*(18|20)\s*,\s*false\s*>)")
    assert flag.search(dots["risk"]) and not flag.search(dots["mean"])


def test_graph_replay_equals_eager():
    for dist in ("categorical", "quantile"):
        kw = dict(ALL, distribution=dist, risk_measure="cvar")
        ga, ea = _agent(**kw), _agent(cuda_graph=False, **kw)
        gm, em = _memory(**MEM_ALL), _memory(**MEM_ALL)
        for step in range(8):
            for ag, mem in ((ga, gm), (ea, em)):
                ag.reset_noise()
                ag.learn(mem)
            assert_bits_equal(cpu(ga.last_loss), cpu(ea.last_loss), f"{dist}: loss of update {step}")
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
    kw = dict(augment_shift=4, risk_measure="wang", risk_eta=-0.5)
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
    assert (hp["risk_measure"], hp["risk_eta"]) == ag.risk == ("wang", -0.5)
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
    assert not any(k.startswith("risk") for k in hp)
    ag.save_checkpoint(str(tmp_path / "r"))
    _refused(ck_agent(seed=8, **kw), None, str(tmp_path / "plain"), match="risk")
    _refused(plain, None, str(tmp_path / "r"), match="risk")
    _refused(ck_agent(seed=8, **dict(kw, risk_eta=0.5)), None, str(tmp_path / "r"), match="risk")
    _refused(ck_agent(seed=8, **dict(kw, risk_measure="cvar", risk_eta=0.5)), None, str(tmp_path / "r"), match="risk")


@pytest.mark.parametrize("case", ["fused-pending", "batch64", "c3", "library-head"])
def test_annealed_horizon_is_the_fixed_horizon(case, monkeypatch):
    """test_gpu_horizon's check as it stands, with both agents built under CVaR."""
    import test_gpu_horizon as TH
    orig = TH._agent
    monkeypatch.setattr(TH, "_agent", lambda seed=5, **kw: orig(seed, **dict(kw, risk_measure="cvar")))
    TH.test_annealed_update_is_the_plain_update_at_its_horizon(case)


@pytest.mark.parametrize("dist", ["categorical", "quantile"])
@pytest.mark.parametrize("measure", ["cvar", "wang"])
def test_acting_and_evaluation_on_the_learners_own_rows(dist, measure):
    """q_select, evaluate_q_batch and the act graph against the reference Q_beta arg-max / max of the head rows the
    learner itself computes for the same states."""
    kw = dict(architecture="data-efficient", hidden_size=64, distribution=dist, risk_measure=measure)
    ag = _agent(**kw)
    val, _ = synthetic_ring(256, seed=4)
    states = val.iter_states(0, 16)
    on = ag.online_net
    sup = None if dist == "quantile" else ag.q_support

    def reference(s):
        with torch.no_grad():
            z = on.head().forward(on.features_nograd(s).contiguous())[0].clone()
        return RR.select_values(z, ag.action_space, ag.atoms, *ag.risk, support=sup)

    Qv, err = reference(states)
    v = ag.evaluate_q_batch(states)
    a, _ = ag.q_select(states)
    assert bool(RR.astar_ok(Qv, err, a).all())
    R.assert_within("max Q_beta", v, Qv.max(1).values, 2 * err.max(1).values, 1.0)
    mean = _agent(**dict(kw, risk_measure=None))
    assert not torch.equal(mean.evaluate_q_batch(states), v), "evaluation reports max Q_beta, not the mean"
    for i in range(4):
        Qi, ei = reference(states[i:i + 1])
        act = ag.act(states[i])
        assert bool(RR.astar_ok(Qi, ei, torch.tensor([act])).all()), "the act graph selects by Q_beta"
        R.assert_within("evaluate_q", torch.tensor([ag.evaluate_q(states[i])], device=DEV), Qi.max(1).values,
                        2 * ei.max(1).values, 1.0)


def test_library_fallback_matches_the_kernel_rows():
    """q_select's torch fallback (shapes the fused head does not take) computes Q_beta within the bound."""
    from rainbow_b200.agent import risk_values
    M, A, Z = 16, 6, 51
    z = (torch.randn(M, Z + A * Z, generator=torch.Generator().manual_seed(2)) * 2).to(DEV)
    x = RR.dueling32(z, A, Z)
    sup = torch.linspace(-10, 10, Z, device=DEV)
    for measure, eta in MEASURES:
        Qv, err = RR.select_values(z, A, Z, measure, eta, sup)
        got = risk_values(torch.softmax(x, -1), measure, eta, support=sup)
        R.assert_within("fallback", got, Qv, err + 1e-5, 1.0)


# ---- whole updates against float64 -----------------------------------------------------------------------------------------
RISK_CASES = [
    _row("categorical", "none", "fixed", "adam", "hard", "off", "off", "off", 32, "fused", "c-h512", "pending"),
    _row("quantile", "none", "fixed", "adam", "hard", "off", "off", "on", 32, "fused", "de-h256", "pending"),
    _row("categorical", "none", "fixed", "adam", "hard", "off", "off", "on", 32, "library", "c-h64", "flushed"),
    _row("quantile", "intensity", "annealed", "adamw", "polyak", "on", "on", "on", 32, "fused", "de-h256", "pending"),
]


@pytest.mark.parametrize("c", RISK_CASES, ids=[case_id(c) for c in RISK_CASES])
def test_update_trajectory_against_float64(c, tmp_path, monkeypatch):
    """test_gpu_update_f64's trajectory check as it stands, with args.risk_measure = "cvar" (eta 0.25) and the double-DQN
    arg-max read by tests/risk_ref.py on the learner's own online s' rows (its ties: the actions risk_ref.astar_ok
    accepts)."""
    import test_gpu_update_f64 as TU
    kwargs = TU.agent_kwargs

    def agent_kwargs(case):
        return dict(kwargs(case), risk_measure="cvar")

    def argmax_choices(q, L, dist, support=None):
        if dist == "quantile":
            Qv, err = RR.quantile_values(q, L, "cvar", 0.25)
        else:
            Qv, err = RR.categorical_values(q, L, support, "cvar", 0.25)
        B, A = Qv.shape
        best = Qv.argmax(1)
        ok = torch.stack([RR.astar_ok(Qv, err, torch.full((B,), a, dtype=torch.long, device=Qv.device))
                          for a in range(A)], 1)
        ties = [(i, torch.nonzero(ok[i]).view(-1).tolist()) for i in torch.nonzero(ok.sum(1) > 1).view(-1).tolist()]
        return best, ties

    monkeypatch.setattr(TU, "agent_kwargs", agent_kwargs)
    monkeypatch.setattr(TU.U, "argmax_choices", argmax_choices)
    TU.test_update_trajectory_against_float64(c, tmp_path, monkeypatch)
