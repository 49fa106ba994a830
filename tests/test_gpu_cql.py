"""CQL(H)'s regulariser on the H100: rb_cql_grad and rb_cql_dueling_grad per element against tests/cql_ref.py over the grid
(Z 2 / 51 / 64 / 65 / 101 / 128 across the R = 2 / 4 boundary, A 1 / 6 / 18, M 1 / 2 / 4, B 1 / 32 / 33 / 512, both heads)
with guard rows and a non-zero incoming gradient; eager launches against graph replay bitwise; refused calls; and the
learner: the update graph's node count, the losses and priorities (the TD loss's, bitwise), eager against replay, resume
and the checkpoint's refusals, whole-update trajectories against float64 (test_gpu_update_f64's check with the
regulariser's gradient added to the float64 objective) and an offline run from a fixed replay."""
import json

import numpy as np
import pytest
import torch

import cql_ref as CQ
from helpers import assert_bits_equal
from test_gpu_augment import update_graph
from test_gpu_parity import DEV, FakeEnv, cpu, make_args, synthetic_ring
from update_cases import _row, case_id

pytestmark = pytest.mark.gpu

GUARD = 3
SENTINEL = 1234.5
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


def run(inp, dz0, gap=True, alpha=None):
    """One launch into a copy of dz0 (fp32, M B rows) with GUARD sentinel rows past it and past gap_out: (rc, out, gap)."""
    n = inp["M"] * inp["B"]
    shape = inp["rows"].shape[1:]
    out = torch.full((n + GUARD,) + tuple(shape), SENTINEL, device=DEV)
    out[:n] = dz0.to(DEV)
    g = torch.full((inp["B"] + GUARD,), SENTINEL, device=DEV)
    rows, acts, w = inp["rows"].to(DEV), inp["actions"].to(DEV), inp["weights"].to(DEV)
    sup = None if inp["support"] is None else inp["support"].to(DEV)
    fn = lib().rb_cql_dueling_grad if inp["entry"] == "dueling" else lib().rb_cql_grad
    rc = fn(rows.data_ptr(), acts.data_ptr(), w.data_ptr(), None if sup is None else sup.data_ptr(),
            inp["alpha"] if alpha is None else alpha, inp["M"], inp["B"], inp["A"], inp["Z"], out.data_ptr(),
            g.data_ptr() if gap else None, stream())
    torch.cuda.synchronize()
    return rc, out, g


GRID = [(1, 1, 1), (6, 2, 32), (18, 4, 33), (6, 1, 512), (18, 2, 512), (1, 4, 32), (18, 1, 1), (6, 4, 33)]


@pytest.mark.parametrize("head", ["categorical", "quantile"])
@pytest.mark.parametrize("entry", ["plain", "dueling"])
@pytest.mark.parametrize("Z", [2, 51, 64, 65, 101, 128])
def test_entries_against_float64(head, entry, Z):
    for A, M, B in GRID:
        inp = CQ.make_inputs(entry, B, A, Z, M, head, seed=Z * 7 + A + M * 3 + B, alpha=2.5,
                             support="0to20" if B == 33 else "pm10")
        dz0 = (torch.randn(inp["rows"].shape, generator=torch.Generator().manual_seed(B + Z)) * 1e-3).float()
        rc, out, gap = run(inp, dz0)
        assert rc == 0, lib().rb_last_error().decode()
        n = M * B
        ref, e_ref, gref, e_gap = CQ.reference(inp, dz0)
        got = out[:n].double().cpu()
        bad = (got - ref).abs() > e_ref
        assert not bool(bad.any()), (A, M, B, float(((got - ref).abs() / e_ref).max()))
        gg = gap[:B].double().cpu()
        assert bool(((gg - gref).abs() <= e_gap).all()), (A, M, B, float(((gg - gref).abs() / e_gap).max()))
        assert bool((out[n:] == SENTINEL).all()) and bool((gap[B:] == SENTINEL).all()), "guard rows untouched"
        _, out2, gap2 = run(inp, dz0, gap=False)
        assert torch.equal(out2, out) and bool((gap2 == SENTINEL).all()), "gap_out is optional"


def test_graph_replay_equals_eager():
    for entry, head in (("dueling", "categorical"), ("plain", "quantile"), ("dueling", "quantile"), ("plain", "categorical")):
        inp = CQ.make_inputs(entry, 33, 18, 51, 2, head, seed=3)
        dz0 = torch.randn(inp["rows"].shape, generator=torch.Generator().manual_seed(2)).float()
        _, eager, egap = run(inp, dz0)
        rows, acts, w = inp["rows"].to(DEV), inp["actions"].to(DEV), inp["weights"].to(DEV)
        sup = None if inp["support"] is None else inp["support"].to(DEV)
        out = torch.empty_like(eager)
        gap = torch.full_like(egap, SENTINEL)
        fn = lib().rb_cql_dueling_grad if entry == "dueling" else lib().rb_cql_grad
        s = torch.cuda.Stream()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            with torch.cuda.graph(graph, stream=s):
                fn(rows.data_ptr(), acts.data_ptr(), w.data_ptr(), None if sup is None else sup.data_ptr(), inp["alpha"],
                   2, 33, 18, 51, out.data_ptr(), gap.data_ptr(), torch.cuda.current_stream().cuda_stream)
        for _ in range(2):
            out.fill_(SENTINEL)
            out[:66] = dz0.to(DEV)
            graph.replay()
            torch.cuda.synchronize()
            assert_bits_equal(cpu(out), cpu(eager), f"{entry} {head}")
            assert_bits_equal(cpu(gap), cpu(egap), f"{entry} {head} gap")


def test_refused_calls_write_nothing():
    for entry in ("plain", "dueling"):
        inp = CQ.make_inputs(entry, 8, 6, 51, 1, "categorical", seed=1)
        dz0 = torch.ones(inp["rows"].shape)
        for alpha in (float("nan"), 0.0, -1.0):
            rc, out, gap = run(inp, dz0, alpha=alpha)
            assert rc != 0 and "alpha" in lib().rb_last_error().decode()
            assert bool((out[:8] == 1).all()) and bool((gap == SENTINEL).all())
        bad = dict(inp, M=9)
        rc, out, gap = run(bad, torch.ones((72,) + tuple(inp["rows"].shape[1:])))
        assert rc != 0 and bool((out[:72] == 1).all()) and bool((gap == SENTINEL).all())


# ---- the learner -----------------------------------------------------------------------------------------------------------
CQL = dict(cql_alpha=1.0)


def _agent(seed=5, **kw):
    from rainbow_b200.agent import Agent
    torch.manual_seed(seed)
    return Agent(make_args(**kw), FakeEnv(6))


def _memory(**args):
    mem, _ = synthetic_ring(CAP, seed=3, args=args)
    mem.seed = 99
    return mem


@pytest.mark.parametrize("head", ["fused-b32", "fused-b64", "library", "quantile", "drq"])
def test_update_graph_nodes(head, tmp_path, monkeypatch):
    kw = {"fused-b64": dict(batch_size=64), "library": dict(fused_head=False), "fused-b32": dict(),
          "quantile": dict(distribution="quantile"), "drq": dict(augment_m=2, augment_k=2, augment_shift=4)}[head]
    names = {}
    for tag, extra in (("none", dict()), ("off", dict(cql_alpha=0.0)), ("on", CQL)):
        names[tag] = update_graph(_agent(**kw, **extra), _memory(), tmp_path / f"{tag}.dot", monkeypatch)
    own = lambda ks: [k for k in ks if k.startswith("k_")]
    cql = "k_cql" if head == "library" else "k_cql_dueling"
    assert names["off"] == names["none"], "off: the same graph"
    assert len(names["on"]) == len(names["none"]) + 1, "one more node"
    assert own(names["on"]).count(cql) == 1
    assert [k for k in names["on"] if k != cql] == names["none"]


@pytest.mark.parametrize("extra", [dict(), dict(fused_head=False), dict(distribution="quantile"),
                                   dict(augment_m=2, augment_k=2, augment_shift=4)])
def test_losses_and_priorities_stay_the_td_loss(extra):
    """The same first update with alpha on and off: the losses and the priorities written back are bitwise equal; the
    parameters move differently; with the key 0 everything equals an agent built without it."""
    runs = {}
    for tag, kw in (("none", dict()), ("zero", dict(cql_alpha=0)), ("on", dict(cql_alpha=3.0))):
        ag, mem = _agent(cuda_graph=False, **extra, **kw), _memory()
        ag.reset_noise()
        ag.learn(mem)
        torch.cuda.synchronize()
        runs[tag] = (cpu(ag.last_loss), cpu(mem.transitions.tree), cpu(ag.optimiser.flat_param),
                     None if ag.last_cql_gap is None else cpu(ag.last_cql_gap))
    for i, what in enumerate(("loss", "priorities", "parameters")):
        assert_bits_equal(runs["zero"][i], runs["none"][i], what)
    assert_bits_equal(runs["on"][0], runs["none"][0], "loss")
    assert_bits_equal(runs["on"][1], runs["none"][1], "priorities")
    assert not np.array_equal(runs["on"][2], runs["none"][2]), "the regulariser moves the parameters"
    assert runs["none"][3] is None and runs["on"][3] is not None
    assert np.isfinite(runs["on"][3]).all() and (runs["on"][3] >= 0).all()


@pytest.mark.parametrize("head", ["fused", "library", "munchausen"])
def test_graph_replay_equals_eager_in_the_learner(head):
    kw = dict(CQL, augment_shift=4, target_tau=0.005, learn_stats=8)
    if head == "library":
        kw["fused_head"] = False
    if head == "munchausen":
        kw.update(distribution="quantile", munchausen=True)
    ga, ea = _agent(**kw), _agent(cuda_graph=False, **kw)
    gm, em = _memory(), _memory()
    for step in range(6):
        for ag, mem in ((ga, gm), (ea, em)):
            ag.reset_noise()
            ag.learn(mem)
        assert_bits_equal(cpu(ga.last_loss), cpu(ea.last_loss), f"loss of update {step}")
        assert_bits_equal(cpu(ga.last_cql_gap), cpu(ea.last_cql_gap), f"gap of update {step}")
    assert ga._graphs and not ea._graphs
    for k in ("flat_param", "exp_avg", "exp_avg_sq"):
        assert_bits_equal(cpu(getattr(ga.optimiser, k)), cpu(getattr(ea.optimiser, k)), k)


def test_resume_equals_never_stopping_and_a_mismatch_is_refused(tmp_path):
    from test_gpu_checkpoint import _agent as ck_agent
    from test_gpu_checkpoint import _assert_same, _before_update, _fresh_memory, _refused, _state, _update
    from test_gpu_checkpoint import _memory as ck_memory
    kw = dict(augment_shift=4, cql_alpha=0.5)
    total, save_at = 8, 3
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
    assert hp["cql_alpha"] == 0.5
    ag, mem = ck_agent(seed=77, **kw), _fresh_memory()
    ag.load_checkpoint(str(tmp_path / "ck"), mem)
    for step in range(save_at, total):
        if step > save_at:
            _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _assert_same(run_a, _state(ag, mem, losses))

    plain = ck_agent(augment_shift=4)
    plain.save_checkpoint(str(tmp_path / "plain"))
    assert "cql_alpha" not in json.load(open(tmp_path / "plain" / "rank0" / "manifest.json"))["hyper_parameters"]
    ag.save_checkpoint(str(tmp_path / "on"))
    _refused(ck_agent(seed=8, **kw), None, str(tmp_path / "plain"), match="cql_alpha")
    _refused(plain, None, str(tmp_path / "on"), match="cql_alpha")
    _refused(ck_agent(seed=8, augment_shift=4, cql_alpha=2.0), None, str(tmp_path / "on"), match="cql_alpha")


def test_offline_training_from_a_fixed_replay():
    """A replay filled once through append from a seeded synthetic dataset whose behaviour policy is a function of the
    state (each frame marks the action taken in it), sampled uniformly (priority_exponent = 0), then a few hundred CQL
    updates with no acting: the mean gap falls and nothing is non-finite."""
    from rainbow_b200.memory import ReplayMemory
    args = make_args(priority_exponent=0.0, batch_size=32, architecture="data-efficient", hidden_size=64, cql_alpha=2.0,
                     learning_rate=1e-3)
    A, cap = 6, 2048
    mem = ReplayMemory(args, cap)
    rs = np.random.RandomState(11)
    for t in range(cap):
        a = int(rs.randint(0, A))
        frame = rs.uniform(0.0, 0.2, (4, 84, 84)).astype(np.float32)
        frame[-1, a * 14:(a + 1) * 14, :] += 0.8
        mem.append(torch.from_numpy(frame).to(DEV), a, float(rs.randint(-1, 2)), bool(rs.uniform() < 0.02))
    torch.manual_seed(5)
    from rainbow_b200.agent import Agent
    ag = Agent(args, FakeEnv(A))
    gaps = []
    for step in range(400):
        ag.learn(mem)
        gaps.append(ag.last_cql_gap.mean())
    torch.cuda.synchronize()
    gaps = torch.stack(gaps).cpu().numpy()
    assert np.isfinite(gaps).all() and np.isfinite(cpu(ag.optimiser.flat_param)).all()
    assert np.isfinite(cpu(ag.last_loss)).all()
    first, last = gaps[:20].mean(), gaps[-20:].mean()
    print(f"\nmean CQL gap: first 20 updates {first:.4f}, last 20 {last:.4f}")
    assert last < 0.5 * first


# ---- whole updates against float64 -----------------------------------------------------------------------------------------
class _AddGrad(torch.autograd.Function):
    """Identity forward; the backward adds `extra` to the incoming gradient."""

    @staticmethod
    def forward(ctx, q, extra):
        ctx.extra = extra
        return q.view_as(q)

    @staticmethod
    def backward(ctx, g):
        return g + ctx.extra, None


def _cql_terms(q, batch, M, alpha):
    """(g, scale) [M B][A][Z] of the regulariser on the float64 online rows of s: cql_ref's gradient, and a scale that
    bounds the fp32 kernel's error over update_ref.TAU_G: the terms' magnitudes times 1 + 2 x the spread of the values
    (sigma's sensitivity to the rounding of Q)."""
    sup = batch.get("support")
    sup = None if "kappa" in batch else sup.double()
    g, _, sigma, Q, p = CQ.grad_logits(q, batch["actions"].long(), batch["weights"].double(), sup, alpha, M)
    B = batch["actions"].shape[0]
    act = batch["actions"].long().repeat(M)
    c = (alpha * batch["weights"].double().repeat(M) / (M * B)).abs().unsqueeze(1)
    amp = sigma + torch.nn.functional.one_hot(act, q.shape[1]).double()
    if sup is None:
        spread = 1 + 2 * q.abs().amax((1, 2), keepdim=True)
        s = (c * amp / q.shape[2]).unsqueeze(2) * spread
        return g, s.expand_as(q)
    spread = 1 + 2 * float(sup.abs().max())
    return g, (c * amp).unsqueeze(2) * p * (sup.abs().view(1, 1, -1) + Q.abs().unsqueeze(2)) * spread


def _with_cql(monkeypatch, alpha=0.8):
    """test_gpu_update_f64's trajectory check with args.cql_alpha set: the float64 update's online rows of s carry the
    regulariser's gradient (and its scale into the per-element bound) through update_ref's own backward."""
    import munchausen_update_ref as MU
    import test_gpu_update_f64 as TU
    import update_ref as U
    cur = {}
    kwargs = TU.agent_kwargs
    monkeypatch.setattr(TU, "agent_kwargs", lambda case: dict(kwargs(case), cql_alpha=alpha))
    a32 = float(np.float32(alpha))

    def wrap(fn):
        def f(*a, **k):
            cur.update(batch=a[9], M=k.get("M", a[11] if len(a) > 11 else 1))
            return fn(*a, **k)
        return f
    monkeypatch.setattr(U, "update_ref", wrap(U.update_ref))
    monkeypatch.setattr(MU, "update_ref", wrap(MU.update_ref))
    orig = U.net_f64

    def net_f64(net, P, f, x, masks=None, hidden_masks=None, absolute=False, keep=None):
        q = orig(net, P, f, x, masks, hidden_masks, absolute=absolute, keep=keep)
        if keep is None and not absolute:
            return q
        n = cur["M"] * cur["batch"]["actions"].shape[0]
        if not absolute:
            g, s = _cql_terms(q.detach()[:n], cur["batch"], cur["M"], a32)
            cur["scale"] = s
            extra = torch.zeros_like(q)
            extra[:n] = g
        else:
            extra = torch.zeros_like(q)
            extra[:n] = cur["scale"][:q.shape[0]]
        return _AddGrad.apply(q, extra)
    monkeypatch.setattr(U, "net_f64", net_f64)
    return TU


TRAJ = {
    "projection": _row("categorical", "none", "fixed", "adam", "hard", "off", "off", "on", 32, "fused", "c-h512",
                       "pending"),
    "projection-library": _row("categorical", "shift", "fixed", "adam", "polyak", "off", "off", "off", 32, "library",
                               "c-h64", "flushed"),
    "quantile": _row("quantile", "none", "fixed", "adam", "hard", "off", "off", "on", 64, "fused", "de-h256", "pending"),
    "c51-drq": _row("categorical", "drq", "fixed", "adam", "polyak", "off", "off", "off", 32, "fused", "c-h512",
                    "flushed"),
}


@pytest.mark.parametrize("name", TRAJ)
def test_update_trajectory_against_float64(name, tmp_path, monkeypatch):
    TU = _with_cql(monkeypatch)
    TU.test_update_trajectory_against_float64(TRAJ[name], tmp_path, monkeypatch)


@pytest.mark.parametrize("name", ["hl_gauss", "two_hot", "munchausen", "qr_drq", "cvar"])
def test_update_trajectory_against_float64_with_the_other_targets(name, tmp_path, monkeypatch):
    """The trajectory checks of the other targets' own test files, as they stand, with the regulariser added."""
    import test_gpu_hl_gauss as HG
    import test_gpu_munchausen as MG
    import test_gpu_qr_drq as QD
    import test_gpu_risk as RG
    import test_gpu_two_hot as TG
    mod, cases = {"hl_gauss": (HG, HG.HLG_CASES), "two_hot": (TG, [c for c, vt in TG.TH_CASES if not vt]),
                  "munchausen": (MG, MG.MUNCH_CASES), "qr_drq": (QD, QD.QR_DRQ_CASES),
                  "cvar": (RG, RG.RISK_CASES)}[name]
    _with_cql(monkeypatch)
    if name == "two_hot":
        mod.test_update_trajectory_against_float64(cases[0], False, tmp_path, monkeypatch)
    else:
        mod.test_update_trajectory_against_float64(cases[0], tmp_path, monkeypatch)
