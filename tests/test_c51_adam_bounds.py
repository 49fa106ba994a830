"""Where the bounds of tests/test_gpu_c51_f64.py and tests/test_gpu_clip_adam_f64.py come from (CPU only).

1. The float64 references are pinned to upstream: c51_ref reproduces the distributional loss the reference recorded
   (tests/golden/learn.npz: m, loss, gradient, a*) within its bound, and adam_ref is torch.nn.utils.clip_grad_norm_ +
   torch.optim.Adam run in float64.
2. Each bound is at least 5x above what fp32 arithmetic makes of the same operation: for the loss, the CPU oracle
   (oracle/rb_oracle.c orc_c51, the kernel's operations in sequential order) on every case of the GPU grid, and a
   sequential fp32 expectation for the arg-max; for Adam the oracle (orc_clip_adam) and a model of k_clip_adam's own
   operations (fp32 FMAs, double-precision bias corrections) with sqrt.approx.f32 and rcp.approx.f32 pushed to the
   error bound the PTX ISA states for them (relative 2^-23 for sqrt; 1 ulp, at most 2^-23 relative, for rcp).
3. Each bound is at least 5x below the error of each semantic slip the GPU tests are meant to catch, on inputs where the
   slip matters (a dropped fix-up, a missing clamp, a tie won by the last action, the dueling mean or 1/A left out, a
   truncated support; an element left unupdated, a step counted while gated, the clip not clamped to 1, grad_scale
   left out of the norm, bias correction one step behind)."""
import numpy as np
import pytest
import torch

import adam_ref as AR
import c51_ref as C
import head_ref as R
import oracle
from helpers import golden, manifest

SLIP_MARGIN = 5


def _ratio(got, ref, scale):
    return R.err_ratio(torch.as_tensor(got), ref, scale, 0.0)[0]


# ---------------------------------------------------------------------------------------------------------------------
# 1. the references against upstream
@pytest.mark.parametrize("case", manifest()["learn_cases"], ids=lambda c: c["name"])
def test_c51_ref_reproduces_the_reference_goldens(case):
    g = golden("learn")
    p = case["name"] + "_"
    t = lambda k: torch.from_numpy(np.ascontiguousarray(g[p + k]))
    B, A, Z = case["B"], case["A"], case["Z"]
    inp = dict(entry="plain", B=B, A=A, Z=Z, support=t("support"), vmin=case["V_min"], vmax=case["V_max"],
               dz=case["delta_z"], gamma_n=case["discount"] ** case["n"], actions=t("actions"), returns=t("returns"),
               nonterminals=t("nonterm"), weights=t("weights"), q_on_s=t("q_s"), q_on_ns=t("q_ns"), q_tg_ns=t("q_t"))
    astar = t("astar")
    ev, evs = C.expected_values(inp)
    assert bool(C.astar_ok(ev, evs, astar).all()) and bool(C.first_of_identical(inp, astar).all())
    m_ref, m_scale = C.projection(inp, astar)
    R.assert_within("m", t("m"), m_ref, m_scale, C.TAU)
    (l_ref, l_scale), (g_ref, g_scale) = C.loss_grad(inp, t("m"))
    R.assert_within("loss", t("loss"), l_ref, l_scale, C.TAU)
    grad = t("grad")
    taken = torch.zeros(B, A, dtype=torch.bool)
    taken[torch.arange(B), inp["actions"]] = True
    assert bool((grad[~taken] == 0).all())
    R.assert_within("grad", grad[taken], g_ref, g_scale, C.TAU)


F32 = lambda x: float(np.float32(x))
ADAM_SETTINGS = [  # (step_count, grad_scale, clip factor max_norm / ||g s||, betas, eps, lr)
    (0, 1.0, 0.1, (0.9, 0.999), 1.5e-4, 6.25e-5), (9, 0.5, 10.0, (0.9, 0.999), 1e-8, 1e-3),
    (10 ** 6, 0.125, 1.0, (0.5, 0.9), 1e-8, 1e-3), (9, 1.0, 0.5, (0.5, 0.9), 1.5e-4, 1e-3)]


def _adam_state(P, step0, seed, gmag=1.0):
    rs = np.random.RandomState(seed)
    p = (rs.standard_normal(P) * 0.01).astype(np.float32)
    p[::7] = 0
    g = (rs.standard_normal(P) * gmag).astype(np.float32)
    m = (rs.standard_normal(P) * 0.3 * gmag * (step0 > 0)).astype(np.float32)
    v = ((rs.uniform(0.5, 1.5, P)) * gmag ** 2 * (step0 > 0)).astype(np.float32)
    return p, g, m, v


@pytest.mark.parametrize("setting", ADAM_SETTINGS, ids=lambda s: f"t{s[0]}-s{s[1]:g}-clip{s[2]:g}-b{s[3][0]:g}")
def test_adam_ref_is_torch_clip_and_adam_in_float64(setting):
    step0, gs, clipf, (b1, b2), eps, lr = setting
    b1, b2, eps, lr = F32(b1), F32(b2), F32(eps), F32(lr)          # what the kernel is passed, exactly
    p, g, m, v = (torch.from_numpy(a) for a in _adam_state(1000, step0, 1))
    max_norm = F32(clipf * float((g.double() * gs).norm()))
    ref = AR.clip_adam(p, g, m, v, step0, gs, max_norm, lr, b1, b2, eps)
    w = torch.nn.Parameter(p.double().clone())
    opt = torch.optim.Adam([w], lr=lr, betas=(b1, b2), eps=eps)
    if step0:
        opt.state[w] = dict(step=torch.tensor(float(step0)), exp_avg=m.double().clone(), exp_avg_sq=v.double().clone())
    w.grad = g.double() * gs
    norm = torch.nn.utils.clip_grad_norm_([w], max_norm)
    opt.step()
    st = opt.state[w]
    assert abs(float(norm) - ref["norm"][0]) <= 1e-13 * ref["norm"][0]
    for name, got in (("p", w.detach()), ("m", st["exp_avg"]), ("v", st["exp_avg_sq"])):
        torch.testing.assert_close(got, ref[name][0], rtol=1e-12, atol=1e-300)


# ---------------------------------------------------------------------------------------------------------------------
# 2. the bounds against fp32 arithmetic
def _fp32_q(inp, which):
    """The logits in fp32 as the kernel forms them (dueling: the sequential fp32 mean of the kernel)."""
    if inp["entry"] == "plain":
        return inp[{"s": "q_on_s", "ns": "q_on_ns", "t": "q_tg_ns"}[which]]
    B, A, Z = inp["B"], inp["A"], inp["Z"]
    z = {"s": inp["z_on"][:B], "ns": inp["z_on"][B:], "t": inp["z_tg"]}[which]
    zv, za = z[:, :Z].unsqueeze(1), z[:, Z:].reshape(-1, A, Z)
    acc = torch.zeros_like(za[:, 0])
    for a in range(A):
        acc = acc + za[:, a]
    return zv + za - (acc / A).unsqueeze(1)


def _ev_fp32(q, support):
    """Expected values of softmax rows in fp32, every sum sequential (the oracle's order)."""
    q = q.numpy().astype(np.float32)
    s = support.numpy().astype(np.float32)
    e = np.exp((q - q.max(-1, keepdims=True)).astype(np.float32)).astype(np.float32)
    tot = np.zeros(q.shape[:-1], np.float32)
    for z in range(q.shape[-1]):
        tot = (tot + e[..., z]).astype(np.float32)
    pz = (e / tot[..., None]).astype(np.float32)
    ev = np.zeros(q.shape[:-1], np.float32)
    for z in range(q.shape[-1]):
        ev = (ev + (s[z] * pz[..., z]).astype(np.float32)).astype(np.float32)
    return torch.from_numpy(ev)


def _oracle_run(inp):
    n = lambda t: t.numpy()
    q = [n(_fp32_q(inp, w).contiguous()) for w in ("s", "ns", "t")]
    loss, grad, m, astar = oracle.c51(*q, n(inp["actions"]), n(inp["returns"]), n(inp["nonterminals"]), n(inp["weights"]),
                                      n(inp["support"]), inp["vmin"], inp["vmax"], inp["dz"], inp["gamma_n"])
    return torch.from_numpy(loss), torch.from_numpy(grad), torch.from_numpy(m), torch.from_numpy(astar)


def test_c51_bounds_are_5x_above_fp32_arithmetic():
    worst = dict(ev=0.0, m=0.0, loss=0.0, grad=0.0)
    for entry in ("plain", "dueling"):
        for B, A, Z, sup in C.CASES:
            inp = C.make_inputs(entry, B, A, Z, sup, seed=B * 1000 + A * 10 + Z)
            loss, grad, m, astar = _oracle_run(inp)
            ev, evs = C.expected_values(inp)
            worst["ev"] = max(worst["ev"], _ratio(_ev_fp32(_fp32_q(inp, "ns"), inp["support"]), ev, evs))
            assert bool(C.astar_ok(ev, evs, astar).all()) and bool(C.first_of_identical(inp, astar).all())
            worst["m"] = max(worst["m"], _ratio(m, *C.projection(inp, astar)))
            (l_ref, l_scale), (g_ref, g_scale) = C.loss_grad(inp, m)
            worst["loss"] = max(worst["loss"], _ratio(loss, l_ref, l_scale))
            worst["grad"] = max(worst["grad"], _ratio(grad[torch.arange(B), inp["actions"]], g_ref, g_scale))
    assert SLIP_MARGIN * worst["ev"] <= C.TAU_EV, worst
    for k in ("m", "loss", "grad"):
        assert SLIP_MARGIN * worst[k] <= C.TAU, (k, worst)


def _fma(a, b, c):
    """fp32 fmaf: the product is exact in float64, one rounding of the sum (float64 then float32; the double rounding
    this can add is far below the bounds checked here)."""
    return (a.astype(np.float64) * b + c).astype(np.float32)


def kernel_model(p, g, m, v, step_count, gs, max_norm, lr, b1, b2, eps, sqrt_err=0.0, rcp_err=0.0):
    """k_sqnorm + k_clip_adam in numpy: fp32 where the kernel is fp32, double for the norm and the bias corrections;
    sqrt.approx / rcp.approx as the exact value times (1 + err)."""
    f = np.float32
    gs_, b1_, b2_, eps_ = f(gs), f(b1), f(b2), f(eps)
    a = (g * gs_).astype(np.float32)
    norm = f(np.sqrt(np.sum(a.astype(np.float64) ** 2)))
    c = f(f(max_norm) / f(norm + f(1e-6)))
    coef = f(min(c, f(1.0)) * gs_)
    t = step_count + 1
    step_size = f(float(f(lr)) / (1.0 - float(b1_) ** t))
    bc2_sqrt = f(1.0 / np.sqrt(1.0 - float(b2_) ** t))
    gc = (g * coef).astype(np.float32)
    m1 = _fma((gc - m).astype(np.float32), np.full_like(m, f(1.0) - b1_), m)
    v1 = _fma(v, np.full_like(v, b2_), ((f(1.0) - b2_) * gc * gc).astype(np.float32))
    sq = (np.sqrt(v1.astype(np.float64)) * (1 + sqrt_err)).astype(np.float32)
    denom = _fma(sq, np.full_like(sq, bc2_sqrt), np.full_like(sq, eps_))
    rcp = (1.0 / denom.astype(np.float64) * (1 + rcp_err)).astype(np.float32)
    p1 = _fma((-step_size * m1).astype(np.float32), rcp, p)
    return p1, m1, v1, float(norm)


def _adam_worst(res, ref):
    p1, m1, v1, norm = res
    out = {k: _ratio(torch.from_numpy(x), *ref[k]) for k, x in (("p", p1), ("m", m1), ("v", v1))}
    out["norm"] = abs(norm - ref["norm"][0]) / ref["norm"][1]
    return out


APPROX = 2.0 ** -23       # PTX ISA: sqrt.approx.f32 max relative error 2^-23; rcp.approx.f32 max 1 ulp


def test_adam_bound_is_5x_above_fp32_arithmetic():
    worst = {}
    for i, (step0, gs, clipf, (b1, b2), eps, lr) in enumerate(ADAM_SETTINGS):
        for gmag in (1.0, 1e-20, 1e4):
            p, g, m, v = _adam_state(4096, step0, 10 + i, gmag)
            max_norm = max(clipf * float((g.astype(np.float64) * F32(gs)) @ (g.astype(np.float64) * F32(gs))) ** 0.5, 1e-30)
            if gmag == 1e-20:
                max_norm = 10.0
            ref = AR.clip_adam(*(torch.from_numpy(x) for x in (p, g, m, v)), step0, gs, max_norm, lr, b1, b2, eps)
            runs = [kernel_model(p, g, m, v, step0, gs, max_norm, lr, b1, b2, eps, se, re)
                    for se in (-APPROX, 0.0, APPROX) for re in (-APPROX, 0.0, APPROX)]
            if gs == 1.0:                                        # the oracle has no grad_scale
                po, go, mo, vo = p.copy(), g.copy(), m.copy(), v.copy()
                no = oracle.clip_adam(po, go, mo, vo, max_norm, lr, b1, b2, eps, step0 + 1)
                runs.append((po, mo, vo, no))
            for res in runs:
                for k, r in _adam_worst(res, ref).items():
                    worst[k] = max(worst.get(k, 0.0), r)
    for k, r in worst.items():
        assert SLIP_MARGIN * r <= AR.TAU, (k, worst)


# ---------------------------------------------------------------------------------------------------------------------
# 3. the bounds against semantic slips
def _project_slip(inp, astar, slip):
    """m of c51_ref.projection with one slip of the kernel's projection."""
    Z = inp["Z"]
    q, L = C.logits(inp, "t")
    pt = torch.softmax(q[torch.arange(inp["B"]), astar], -1)
    s = inp["support"].double().unsqueeze(0)
    r, nt = inp["returns"].double().unsqueeze(1), inp["nonterminals"].double().view(-1, 1)
    vmin, vmax, dz, gn = C.f32(inp["vmin"]), C.f32(inp["vmax"]), C.f32(inp["dz"]), C.f32(inp["gamma_n"])
    f = torch.float32                                            # b in the kernel's fp32: where the fix-ups act
    tz = r.to(f) + (nt.to(f) * gn) * s.to(f)
    tz = tz.clamp(max=vmax) if slip == "no_vmin_clamp" else tz.clamp(vmin, vmax)
    b = ((tz - vmin) / dz).double()
    lo, up = b.floor(), b.ceil()
    if slip != "no_fixup_lo":
        lo = torch.where((up > 0) & (lo == up), lo - 1, lo)
    if slip != "no_fixup_up":
        up = torch.where((lo < Z - 1) & (lo == up), up + 1, up)
    wl, wu = pt * (up - b), pt * (b - lo)
    if slip == "fullscan_l_short":                               # the l-side scan never reaches atom Z - 1
        wl[:, Z - 1] = 0
    m = torch.zeros(b.shape[0], Z + 2, dtype=torch.float64)
    ok = lambda k: (k >= 0) & (k < Z)                             # the kernel's gather never visits other indices
    m.scatter_add_(1, torch.where(ok(lo), lo, Z + 1).long(), wl)
    m.scatter_add_(1, torch.where(ok(up), up, Z + 1).long(), wu)
    return m[:, :Z]


@pytest.mark.parametrize("slip,sup,entry", [("no_fixup_lo", "pm10", "plain"), ("no_fixup_up", "pm10", "plain"),
                                            ("no_vmin_clamp", "m3to7", "plain"), ("fullscan_l_short", "rev", "dueling"),
                                            ("tie_to_last", "pm10", "dueling")])
def test_c51_projection_slips_are_5x_above_tau(slip, sup, entry):
    """On a batch holding every row kind: the largest |m_slip - m| / scale is at least 5 TAU."""
    B, A, Z = 35, 6, 51
    inp = C.make_inputs(entry, B, A, Z, sup, seed=7)
    ev, _ = C.expected_values(inp)
    astar = ev.argmax(1)                                         # first maximum, like torch.argmax
    m_ref, m_scale = C.projection(inp, astar)
    if slip == "tie_to_last":
        tied = ~C.first_of_identical(inp, torch.full_like(astar, A - 1))
        assert bool(tied.any())
        last = torch.where(tied, A - 1, astar)
        m_slip = C.projection(inp, last)[0]
    else:
        m_slip = _project_slip(inp, astar, slip)
    assert _ratio(m_slip, m_ref, m_scale) >= SLIP_MARGIN * C.TAU


@pytest.mark.parametrize("slip", ["no_mean", "support64"])
def test_c51_argmax_slips_are_5x_above_tau_ev(slip):
    """The slipped arg-max picks, on some row, an action whose expected value is short of the best by 5 TAU_EV scales."""
    B, A, Z = 35, 6, 128 if slip == "support64" else 51
    inp = C.make_inputs("dueling", B, A, Z, "pm10", seed=8)
    ev, evs = C.expected_values(inp)
    q, L = C.logits(inp, "ns")
    if slip == "no_mean":
        zs = inp["z_on"][B:].double()
        q = zs[:, :Z].unsqueeze(1) + zs[:, Z:].reshape(B, A, Z)
    sup = inp["support"].double().clone()
    if slip == "support64":
        sup[64:] = 0
    a_slip = (torch.softmax(q, -1) * sup).sum(-1).argmax(1)
    best = ev.argmax(1)
    short = (ev.gather(1, best[:, None]) - ev.gather(1, a_slip[:, None])).squeeze(1)
    need = SLIP_MARGIN * C.TAU_EV * (evs.gather(1, best[:, None]) + evs.gather(1, a_slip[:, None])).squeeze(1)
    assert bool((short >= need).any())


def test_c51_dueling_dz_without_inv_a_is_5x_above_tau():
    B, A, Z = 35, 6, 51
    inp = C.make_inputs("dueling", B, A, Z, "pm10", seed=9)
    astar = C.expected_values(inp)[0].argmax(1)
    m = C.projection(inp, astar)[0]
    _, (g, gsc) = C.loss_grad(inp, m)
    dz, dzs = C.dueling_dz(inp, g, gsc)
    sel = torch.zeros(B, A, 1, dtype=torch.float64)
    sel[torch.arange(B), inp["actions"]] = 1.0
    slip = torch.cat([g, (g.unsqueeze(1) * sel).reshape(B, A * Z)], 1)
    assert _ratio(slip, dz, dzs) >= SLIP_MARGIN * C.TAU


def test_mass_dropping_supports_round_past_the_last_atom():
    """The grid's Z 62 V +-1 and Z 100 V +-100 supports put b of Vmax past Z - 1 in fp32 (the kernel then drops
    pt (b - l)); V +-10 at 51 atoms does not."""
    for Z, sup, past in ((62, "pm1", True), (100, "pm100", True), (51, "pm10", False)):
        assert (Z, sup) in {(c[2], c[3]) for c in C.CASES}
        _, vmin, vmax, dz = C.support_of(sup, Z)
        b = np.float32(np.float32(vmax) - np.float32(vmin)) / np.float32(dz)
        assert (b > Z - 1) == past, (Z, sup, b)


@pytest.mark.parametrize("slip", ["last_not_updated", "past_first_round", "step_when_gated", "no_fmin", "norm_without_scale",
                                  "bias_correction_behind"])
def test_adam_slips_are_5x_above_tau(slip):
    step0, gs, b1, b2, eps, lr = 9, 0.5, 0.9, 0.999, 1e-8, 1e-3
    p, g, m, v = (torch.from_numpy(a) for a in _adam_state(4096, step0, 3))
    gnorm = float((g.double() * F32(gs)).norm())
    clipf = 10.0 if slip == "no_fmin" else 0.5
    max_norm = clipf * gnorm
    ref = AR.clip_adam(p, g, m, v, step0, gs, max_norm, lr, b1, b2, eps)
    if slip in ("last_not_updated", "past_first_round"):        # those elements keep their old values
        sl = slice(-1, None) if slip == "last_not_updated" else slice(2048, None)
        worst = _ratio(p[sl], ref["p"][0][sl], ref["p"][1][sl])
    elif slip in ("step_when_gated", "bias_correction_behind"):
        t = step0 + 1 if slip == "step_when_gated" else step0 - 1
        worst = _ratio(AR.clip_adam(p, g, m, v, t, gs, max_norm, lr, b1, b2, eps)["p"][0], *ref["p"])
    elif slip == "no_fmin":
        c = max_norm / (gnorm + 1e-6)                          # > 1: the gradient is scaled up instead of left alone
        worst = _ratio(AR.clip_adam(p, g * c, m, v, step0, gs, 1e30, lr, b1, b2, eps)["m"][0], *ref["m"])
    else:
        worst = abs(gnorm / F32(gs) - ref["norm"][0]) / ref["norm"][1]
    assert worst >= SLIP_MARGIN * AR.TAU, worst
