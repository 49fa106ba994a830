"""Intensity augmentation and DrQ's K / M averaging on the GPU (rb_gather_aug, rb_c51_dueling_avg_loss_grad,
args.augment_intensity / augment_m / augment_k).

* The gather: every copy of every observation equals the numpy shift (philox_ref) of rb_gather's own output at the
  recorded offsets times the recorded multiplier, one fp32 multiply, bitwise; the scalars are rb_gather's; guard rows stay
  untouched; a graph replay equals the eager launch and its node is k_gather_aug.  At M = K = 1 without intensity it equals
  rb_gather_shift bitwise; with intensity on, copy 0's offsets are still rb_gather_shift's.
* The draws: copy j's offsets are philox_ref's with stream word 0x53484654 + j; the multipliers are within
  drq_ref.MULT_TOL of the float64 reference and clamped ones are fma(s, +-2, 1) bitwise; over 10^5 samples the normals
  inside +-2 follow the truncated normal (KS), the clamp fractions are 2 (1 - Phi(2)), copies and sides are uncorrelated,
  and successive batches differ.
* The loss kernel: per element within c51_ref.TAU of drq_ref (tolerance sized in test_drq_host.py), both template
  variants read from the graph's nodes; at M = K = 1 bitwise rb_c51_dueling_loss_grad; with identical copies loss, m and
  a* bitwise those of M = K = 1.
* The learner: identical copies (pad 0, intensity 0, M = K = 2) give a plain agent's loss, m and priorities bitwise and
  its gradient within 5e-7 of its largest element; with distinct copies (C3 and canonical / hidden 64, M = K = 2, shift 4,
  intensity 0.05) the loss, every parameter gradient and the parameters after Adam are held to a float64 DrQ update over
  the update's own gathered rows, and the priorities are fl32(sqrt(loss)) bitwise; seven graph replays equal seven eager updates; the update graph swaps only the gather (and, with
  M or K > 1, the loss kernel); a resumed run equals one that never stopped; learner statistics hold the averaged loss and m and copy 0's q.
* The surface: acting and evaluation are unaugmented; rng="numpy", a foreign memory, the library head with M > 1,
  M B > 512 and out-of-range arguments are refused.
Deterministic cuDNN, like the other trajectory tests."""
import json

import numpy as np
import pytest
import torch

import adam_ref as AR
import c51_ref as C
import drq_ref as D
import philox_ref as P
from helpers import assert_bits_equal
from test_gpu_augment import GUARD, NAN, Outputs, episodic_memory, gather, update_graph
from test_gpu_head_f64 import graph_kernels
from test_gpu_parity import DEV, FakeEnv, cpu, make_args, synthetic_ring
from update_ref import f64_forward, f64_projection

pytestmark = pytest.mark.gpu

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


class AugOutputs:
    """rb_gather_aug's buffers, with GUARD rows past each, prefilled with NaN / -1 / -7."""

    def __init__(self, B, history, M, K):
        self.B, self.M, self.K, self.c = B, M, K, max(M, K)
        self.states = torch.full((M * B + GUARD, history, 84, 84), NAN, device=DEV)
        self.next_states = torch.full((K * B + GUARD, history, 84, 84), NAN, device=DEV)
        self.actions = torch.full((B + GUARD,), -1, dtype=torch.int64, device=DEV)
        self.returns = torch.full((B + GUARD,), NAN, device=DEV)
        self.nonterminals = torch.full((B + GUARD,), NAN, device=DEV)
        n = 2 * self.c * B
        self.shifts_flat = torch.full((2 * n + 8,), -7, dtype=torch.int32, device=DEV)
        self.scales_flat = torch.full((n + 8,), NAN, device=DEV)
        self.shifts = self.shifts_flat[:2 * n].view(2, self.c, B, 2)
        self.scales = self.scales_flat[:n].view(2, self.c, B)

    def host(self):
        B = self.B
        return dict(states=cpu(self.states[:self.M * B]), next_states=cpu(self.next_states[:self.K * B]),
                    actions=cpu(self.actions[:B]), returns=cpu(self.returns[:B]), nonterminals=cpu(self.nonterminals[:B]),
                    shifts=cpu(self.shifts), scales=cpu(self.scales))

    def assert_guards(self):
        B = self.B
        assert torch.isnan(self.states[self.M * B:]).all() and torch.isnan(self.next_states[self.K * B:]).all()
        assert (self.actions[B:] == -1).all() and torch.isnan(self.returns[B:]).all()
        assert torch.isnan(self.nonterminals[B:]).all()
        assert (self.shifts_flat[4 * self.c * B:] == -7).all() and torch.isnan(self.scales_flat[2 * self.c * B:]).all()


def gather_aug(mem, didx, out, pad, intensity, seed, counter):
    tr = mem.transitions
    p = lambda t: t.data_ptr()
    rc = lib().rb_gather_aug(p(tr.frames), p(tr.timestep), p(tr.action), p(tr.reward), p(tr.nonterminal), tr.size, p(didx),
                             out.B, mem.history, mem.n, p(mem.n_step_scaling), p(out.states), p(out.next_states),
                             p(out.actions), p(out.returns), p(out.nonterminals), pad, intensity, out.M, out.K, seed,
                             p(counter), p(out.shifts), p(out.scales), stream())
    assert rc == 0, lib().rb_last_error()


def check_multipliers(scales, seed, c, B, copies, s):
    """The recorded multipliers against drq_ref: within MULT_TOL, clamped ones bitwise, exactly 1 without intensity."""
    if s == 0.0:
        assert (scales == np.float32(1.0)).all()
        return None
    ref, n = D.multipliers(seed, c, B, copies, s)
    assert np.abs(scales.astype(np.float64) - ref).max() <= D.MULT_TOL * s + 2.0 ** -23
    for sign in (1, -1):
        sel = sign * n > 2.0 + 1e-4
        assert (scales[sel] == D.clamp_value(s, sign)).all()
    return n


def expected_copy(x, offsets, mult, pad, s):
    y = P.shift_ref(x, offsets, pad)
    return y if s == 0.0 else (y * mult.astype(np.float32)[:, None, None, None]).astype(np.float32)


# (history, n, B, pad, M, K, intensity)
GATHER_CASES = [(4, 3, 32, 4, 2, 2, 0.05), (4, 3, 32, 4, 1, 1, 0.05), (4, 20, 32, 1, 1, 2, 0.05), (1, 1, 32, 16, 2, 1, 0.5),
                (4, 60, 32, 0, 2, 2, 0.05), (4, 3, 1, 16, 8, 8, 0.05), (4, 3, 512, 4, 2, 2, 0.05), (1, 1, 512, 0, 1, 2, 0.0),
                (4, 60, 512, 16, 1, 1, 0.5), (4, 3, 32, 0, 8, 8, 0.0), (4, 20, 1, 1, 2, 1, 0.0), (4, 3, 512, 1, 8, 8, 0.05)]


@pytest.mark.parametrize("history,n,B,pad,M,K,s", GATHER_CASES,
                         ids=[f"h{h}-n{n}-B{B}-p{p}-M{m}-K{k}-s{s}" for h, n, B, p, m, k, s in GATHER_CASES])
def test_gather_aug_is_the_numpy_augmentation_of_rb_gather(history, n, B, pad, M, K, s, tmp_path):
    mem, ts = episodic_memory(history, n)
    cap = mem.capacity
    rs = np.random.RandomState(B * 131 + pad * 7 + history + n + 1000 * M + 100 * K)
    idx = rs.randint(0, cap, B)
    idx[:min(B, 4)] = [0, 1, cap - 1, 2][:min(B, 4)]
    idx[4:8] = rs.choice(np.flatnonzero(ts == 1), 4)[:max(0, min(B, 8) - 4)]
    didx = torch.from_numpy(idx.astype(np.int64)).to(DEV)
    seed = int(rs.randint(0, 2 ** 62)) * 3 + 1
    c = (int(rs.randint(1, 2 ** 20)) << 32) + int(rs.randint(0, 2 ** 31))
    counter = torch.tensor([c], dtype=torch.int64, device=DEV)
    copies = max(M, K)

    plain, aug = Outputs(B, history), AugOutputs(B, history, M, K)
    gather(mem, didx, plain)
    gather_aug(mem, didx, aug, pad, s, seed, counter)
    torch.cuda.synchronize()
    a, g = plain.host(), aug.host()
    plain.assert_guards()
    aug.assert_guards()
    assert int(counter.item()) == c, "the gather reads the counter, it does not advance it"

    off = D.aug_offsets(seed, c, B, pad, copies)
    assert_bits_equal(g["shifts"], off, "offsets")
    if pad:
        assert_bits_equal(off[:, 0], P.shift_offsets(seed, c, B, pad), "copy 0's offsets are rb_gather_shift's")
    check_multipliers(g["scales"], seed, c, B, copies, s)
    for j in range(M):
        assert_bits_equal(g["states"][j * B:(j + 1) * B], expected_copy(a["states"], off[0, j], g["scales"][0, j], pad, s),
                          f"state copy {j}")
    for k in range(K):
        assert_bits_equal(g["next_states"][k * B:(k + 1) * B],
                          expected_copy(a["next_states"], off[1, k], g["scales"][1, k], pad, s), f"next-state copy {k}")
    for key in ("actions", "returns", "nonterminals"):
        assert_bits_equal(g[key], a[key], key)

    replay = AugOutputs(B, history, M, K)
    _, _, dot = graph_kernels(lambda: gather_aug(mem, didx, replay, pad, s, seed, counter), tmp_path / "gather.dot")
    assert "k_gather_aug" in dot
    r = replay.host()
    for key in g:
        assert_bits_equal(r[key], g[key], "graph replay: " + key)
    replay.assert_guards()


@pytest.mark.parametrize("pad", [1, 4, 16])
def test_one_copy_without_intensity_is_rb_gather_shift(pad):
    history, n, B = 4, 3, 64
    mem, _ = episodic_memory(history, n)
    didx = torch.randint(0, mem.capacity, (B,), device=DEV)
    counter = torch.tensor([(3 << 32) + 5], dtype=torch.int64, device=DEV)
    sh, aug = Outputs(B, history), AugOutputs(B, history, 1, 1)
    gather(mem, didx, sh, pad, 77, counter)
    gather_aug(mem, didx, aug, pad, 0.0, 77, counter)
    torch.cuda.synchronize()
    a, g = sh.host(), aug.host()
    for key in ("states", "next_states", "actions", "returns", "nonterminals"):
        assert_bits_equal(g[key], a[key], key)
    assert_bits_equal(g["shifts"][:, 0], a["shifts"], "offsets")
    assert (g["scales"] == np.float32(1.0)).all()


def test_draws_follow_the_streams_and_are_distributed_as_stated():
    from scipy import stats
    from rainbow_b200.memory import _SampleWorkspace
    mem, _ = synthetic_ring(65536, seed=2)
    mem.seed = 0x9E3779B97F4A7C15
    B, rounds, s, pad = 2048, 50, 0.05, 4
    ws = _SampleWorkspace(B, mem.history, mem.device, (2, 2))
    ns, prev = [], None
    for _ in range(rounds):
        mem.sample_into(ws, shift_pad=pad, intensity=s, copies=(2, 2))
        sh, sc = cpu(ws.shifts).copy(), cpu(ws.scales).copy()
        c = int(mem._rng_counter.item())
        assert_bits_equal(sh, D.aug_offsets(mem.seed, c, B, pad, 2), f"offsets at counter {c}")
        check_multipliers(sc, mem.seed, c, B, 2, s)
        assert prev is None or not np.array_equal(sc, prev), "successive batches draw afresh"
        prev = sc
        ns.append((sc.astype(np.float64) - 1.0) / float(np.float32(s)))
    n = np.concatenate(ns, axis=2)                          # [2][2][rounds * B]
    N = n.shape[2]
    clamp = 2 * stats.norm.sf(2.0)
    for side in (0, 1):
        for j in (0, 1):
            x = n[side, j]
            inside = x[np.abs(x) < 1.999]
            assert stats.kstest(inside, stats.truncnorm(-1.999, 1.999).cdf).pvalue > 1e-4
            frac = float((np.abs(x) > 1.9999).mean())
            assert abs(frac - clamp) < 5 * np.sqrt(clamp * (1 - clamp) / N), frac
    for a, b in (((0, 0), (1, 0)), ((0, 0), (0, 1)), ((1, 0), (1, 1)), ((0, 1), (1, 1))):
        assert abs(np.corrcoef(n[a], n[b])[0, 1]) < 5 / np.sqrt(N), (a, b)


# ---- the loss kernel -------------------------------------------------------------------------------------------------------
def run_avg(inp, m_out=True):
    B, A, Z, M, K = inp["B"], inp["A"], inp["Z"], inp["M"], inp["K"]
    loss = torch.full((B,), NAN, device=DEV)
    dz = torch.full((M * B, Z + A * Z), NAN, device=DEV)
    m = torch.full((B, Z), NAN, device=DEV)
    astar = torch.full((K, B), -1, dtype=torch.int64, device=DEV)
    p = lambda t: t.data_ptr()
    rc = lib().rb_c51_dueling_avg_loss_grad(p(inp["z_on"]), p(inp["z_tg"]), A, Z, p(inp["actions"]), p(inp["returns"]),
                                            p(inp["nonterminals"]), p(inp["weights"]), p(inp["support"]), inp["vmin"],
                                            inp["vmax"], inp["dz"], inp["gamma_n"], B, M, K, p(loss), p(dz),
                                            p(m) if m_out else None, p(astar), stream())
    assert rc == 0, lib().rb_last_error()
    return dict(loss=loss, dz=dz, m=m, astar=astar)


def run_plain(inp):
    B, A, Z = inp["B"], inp["A"], inp["Z"]
    loss, dz = torch.empty(B, device=DEV), torch.empty((B, Z + A * Z), device=DEV)
    m, astar = torch.empty((B, Z), device=DEV), torch.empty(B, dtype=torch.int64, device=DEV)
    p = lambda t: t.data_ptr()
    rc = lib().rb_c51_dueling_loss_grad(p(inp["z_on"]), p(inp["z_tg"]), A, Z, p(inp["actions"]), p(inp["returns"]),
                                        p(inp["nonterminals"]), p(inp["weights"]), p(inp["support"]), inp["vmin"], inp["vmax"],
                                        inp["dz"], inp["gamma_n"], B, p(loss), p(dz), p(m), p(astar), stream())
    assert rc == 0, lib().rb_last_error()
    return dict(loss=loss, dz=dz, m=m, astar=astar.view(1, B))


LOSS_CASES = [(32, 6, 51, "pm10", 2, 2), (5, 1, 2, "pm10", 1, 2), (33, 18, 51, "m3to7", 2, 1), (35, 6, 128, "0to20", 3, 2),
              (3, 18, 128, "pm10", 2, 2), (35, 6, 51, "pm10", 8, 8), (512, 6, 51, "pm10", 2, 2), (1, 18, 64, "0to20", 8, 8),
              (40, 1, 101, "0to20", 2, 4)]


@pytest.mark.parametrize("case", LOSS_CASES, ids=[f"B{c[0]}-A{c[1]}-Z{c[2]}-M{c[4]}-K{c[5]}" for c in LOSS_CASES])
def test_avg_loss_against_float64(case, tmp_path):
    B, A, Z, sup, M, K = case
    inp = D.make_inputs(B, A, Z, sup, 11 + B + Z, M, K)
    dev = C.to(inp, DEV)
    _, out, dot = graph_kernels(lambda: run_avg(dev), tmp_path / "avg.dot")
    assert f"k_c51_dueling_avgILi{2 if Z <= 64 else 4}E" in dot
    eager = run_avg(dev)
    torch.cuda.synchronize()
    for k in out:
        assert_bits_equal(cpu(out[k]), cpu(eager[k]), "graph replay: " + k)
    got = {k: v.cpu() for k, v in eager.items()}
    m_ref, m_sc, _, ok = D.target(inp, got["astar"])
    assert ok, "a* within the arg-max's rounding"
    (l_ref, l_sc), _, (dz_ref, dz_sc) = D.loss_dz(inp, got["m"])
    for name, g, ref, sc in (("m", got["m"], m_ref, m_sc), ("loss", got["loss"], l_ref, l_sc),
                             ("dz", got["dz"], dz_ref, dz_sc)):
        err = torch.nan_to_num((g.double() - ref).abs() / sc, nan=0.0)
        assert torch.isfinite(g).all() and float(err.max()) <= C.TAU, f"{name}: {float(err.max()):.3g}"
    zero_w = inp["weights"] == 0
    assert (got["dz"].view(M, B, -1)[:, zero_w] == 0).all()


@pytest.mark.parametrize("B,A,Z", [(32, 6, 51), (35, 18, 128), (1, 1, 2), (512, 6, 51)])
def test_one_copy_is_rb_c51_dueling_loss_grad_and_identical_copies_average_exactly(B, A, Z):
    inp = D.make_inputs(B, A, Z, "pm10", 3 + B, 1, 1)
    dev = C.to(inp, DEV)
    a, b = run_plain(dev), run_avg(dev)
    torch.cuda.synchronize()
    for k in a:
        assert_bits_equal(cpu(b[k]), cpu(a[k]), f"M = K = 1: {k}")
    for M, K in ((2, 2), (1, 2), (2, 1)):   # x + x = 2x and 2x / 2 are exact; a third copy would round
        same = dict(dev, M=M, K=K, z_on=torch.cat([dev["z_on"][:B]] * M + [dev["z_on"][B:]] * K),
                    z_tg=torch.cat([dev["z_tg"]] * K))
        c = run_avg(same)
        torch.cuda.synchronize()
        for k in ("loss", "m"):
            assert_bits_equal(cpu(c[k]), cpu(a[k]), f"identical copies M {M} K {K}: {k}")
        assert_bits_equal(cpu(c["astar"]), np.repeat(cpu(a["astar"]), K, 0), "a*")


# ---- the learner -----------------------------------------------------------------------------------------------------------
def _agent(seed=5, **kw):
    from rainbow_b200.agent import Agent
    torch.manual_seed(seed)
    return Agent(make_args(**kw), FakeEnv(6))


def _memory(**args):
    mem, _ = synthetic_ring(CAP, seed=3, args=args)
    mem.seed = 99
    return mem


DRQ = dict(augment_shift=4, augment_intensity=0.05, augment_m=2, augment_k=2)


def test_identical_copies_equal_a_plain_agent():
    """Pad 0, intensity 0, M = K = 2 writes two identical copies: m = (m0 + m0) / 2 and loss = (l + l) / 2 are exact, the
    gradient of each copy is half the plain one (w / 2B), and the head / conv backward sums the two halves in another
    order -- so loss, m and priorities are bitwise a plain agent's and the gradient agrees to 5e-7 of its largest
    element."""
    for kw in (dict(), dict(architecture="data-efficient", hidden_size=256, multi_step=20)):
        dup, plain = _agent(augment_m=2, augment_k=2, learn_stats=8, cuda_graph=False, **kw), \
            _agent(learn_stats=8, cuda_graph=False, **kw)
        mem_kw = {k: v for k, v in kw.items() if k == "multi_step"}
        md, mp = _memory(**mem_kw), _memory(**mem_kw)
        for ag, mem in ((dup, md), (plain, mp)):
            ag.reset_noise()
            ag.learn(mem)
        torch.cuda.synchronize()
        assert_bits_equal(cpu(dup.last_loss), cpu(plain.last_loss), "loss")
        assert_bits_equal(cpu(dup._stats["last"]["m"]), cpu(plain._stats["last"]["m"]), "m")
        assert_bits_equal(cpu(md.transitions.tree), cpu(mp.transitions.tree), "priorities")
        gd, gp = dup.optimiser.flat_grad.double(), plain.optimiser.flat_grad.double()
        # fp32 sums of the same terms in another order: a few units of 2^-24 of the largest element
        assert float((gd - gp).abs().max()) <= 5e-7 * float(gp.abs().max())


# ---- the DrQ update against float64 ---------------------------------------------------------------------------------------
# Bounds: those of the whole-update comparison of DESIGN.md §4 (loss 1e-5; gradients 1e-6 head / 2e-6 conv; parameters
# after Adam 1e-7 head / 2e-7 conv, all absolute).  The DrQ update runs the same kernels (3xTF32 head, fp32 cuDNN convs,
# fp32 C51, clip + Adam) over (M + K) B = 4B forward and M B = 2B backward rows: every gradient element is a sum of twice
# as many terms, each carrying half the weight (w / (M B)), so the accumulated rounding stays within what the bounds were
# set for at B rows.  The priorities are fl32(loss^omega) = fl32(sqrt(loss)) at omega 0.5, bitwise, like §4's write-back.
TOL = dict(loss=1e-5, grad_head=1e-6, grad_conv=2e-6, param_head=1e-7, param_conv=2e-7)


def _f64_update(ag, ws, before, M, K):
    """The DrQ update in float64 over the update's own gathered rows: (loss [B], {name: grad}, flat parameters after
    clip + Adam)."""
    on, tg, opt = ag.online_net, ag.target_net, ag.optimiser
    B = ws.B
    P = {n: t.double().requires_grad_() for n, t in before["online"].items()}
    T = {n: t.double() for n, t in before["target"].items()}
    q_on = f64_forward(on, P, on.noise_factors(), ws.both_states.double())
    with torch.no_grad():
        q_t = f64_forward(tg, T, tg.noise_factors(), ws.next_states.double())
        r, nt, w = ws.returns.double(), ws.nonterminals.double().view(-1), ws.weights.double()
        sup, rows = ag.support.double(), torch.arange(B, device=ws.actions.device)
        ms = []
        for k in range(K):
            q_ns = q_on[(M + k) * B:(M + k + 1) * B]
            best = (torch.softmax(q_ns, 2) * sup).sum(2).argmax(1)
            ms.append(f64_projection(ag, q_t[k * B:(k + 1) * B][rows, best], r, nt))
        m = sum(ms) / K
    loss = sum(-(m * torch.log_softmax(q_on[j * B:(j + 1) * B][rows, ws.actions], 1)).sum(1) for j in range(M)) / M
    ((w * loss).sum() / B).backward()
    grads = {n: t.grad for n, t in P.items()}
    g = torch.zeros_like(opt.flat_grad, dtype=torch.float64)
    for n, p in on.named_parameters():
        off = (p.data_ptr() - opt.flat_param.data_ptr()) // 4
        g[off:off + p.numel()] = grads[n].reshape(-1)
    ref = AR.clip_adam(before["flat_param"], g, before["exp_avg"], before["exp_avg_sq"], before["step_count"], 1.0,
                       opt.max_norm, opt.lr, opt.betas[0], opt.betas[1], opt.eps)
    return loss.detach(), grads, ref["p"][0]


@pytest.mark.parametrize("kw", [dict(architecture="data-efficient", hidden_size=256, multi_step=20),
                                dict(architecture="canonical", hidden_size=64)], ids=["c3", "canonical-h64"])
def test_drq_update_against_float64(kw):
    """Three updates (two eager warm-ups, then the captured graph) with M = K = 2, shift 4, intensity 0.05: per-sample loss,
    every parameter gradient and the parameters after clip + Adam against _f64_update, within TOL; sum-tree leaves of the
    sampled indices equal fl32(sqrt(loss)) bitwise."""
    ag = _agent(**DRQ, **kw)
    mem = _memory(**{k: v for k, v in kw.items() if k == "multi_step"})
    on, opt = ag.online_net, ag.optimiser
    assert ag._fused_path(ag.batch_size) and mem.priority_exponent == 0.5
    for step in range(3):
        ag.reset_noise()
        torch.cuda.synchronize()
        before = dict(online={n: p.detach().clone() for n, p in on.named_parameters()},
                      target={n: p.detach().clone() for n, p in ag.target_net.named_parameters()},
                      flat_param=opt.flat_param.clone(), exp_avg=opt.exp_avg.clone(), exp_avg_sq=opt.exp_avg_sq.clone(),
                      step_count=int(opt.step_count.item()))
        ag.learn(mem)
        torch.cuda.synchronize()
        ws = mem._last
        assert int(ws.status[0].item()) == 1 and ws.both_states.shape[0] == 4 * ag.batch_size
        assert (cpu(ws.scales) != np.float32(1.0)).any() and (cpu(ws.shifts) != 4).any()
        loss_ref, grads, p_ref = _f64_update(ag, ws, before, 2, 2)
        got = cpu(ag.last_loss)
        assert float((ag.last_loss.double() - loss_ref).abs().max()) <= TOL["loss"], f"loss, update {step}"
        tidx = cpu(ws.tree_idx)
        last = np.array([i for i in range(len(tidx)) if tidx[i] not in tidx[i + 1:]])   # duplicates: the last write wins
        assert_bits_equal(cpu(mem.transitions.tree)[tidx[last]], np.sqrt(got)[last], f"priorities, update {step}")
        for n, p in on.named_parameters():
            conv = n.startswith("convs")
            d = float((p.grad.double() - grads[n]).abs().max())
            assert d <= TOL["grad_conv" if conv else "grad_head"], f"gradient of {n}, update {step}: {d:.3g}"
            off = (p.data_ptr() - opt.flat_param.data_ptr()) // 4
            d = float((p.detach().double().reshape(-1) - p_ref[off:off + p.numel()]).abs().max())
            assert d <= TOL["param_conv" if conv else "param_head"], f"{n} after Adam, update {step}: {d:.3g}"
    assert set(ag._graphs) == {True}


def test_graph_replay_equals_eager():
    ga, ea = _agent(**DRQ), _agent(cuda_graph=False, **DRQ)
    gm, em = _memory(), _memory()
    for step in range(7):
        for ag, mem in ((ga, gm), (ea, em)):
            ag.reset_noise()
            ag.learn(mem)
        assert_bits_equal(cpu(ga.last_loss), cpu(ea.last_loss), f"loss of update {step}")
        assert_bits_equal(cpu(gm._last.scales), cpu(em._last.scales), f"multipliers of update {step}")
    assert ga._graphs and not ea._graphs
    torch.cuda.synchronize()
    for k in ("flat_param", "exp_avg", "exp_avg_sq"):
        assert_bits_equal(cpu(getattr(ga.optimiser, k)), cpu(getattr(ea.optimiser, k)), k)
    assert_bits_equal(cpu(gm.transitions.tree), cpu(em.transitions.tree), "tree")


def test_update_graph_nodes(tmp_path, monkeypatch):
    names = {}
    for tag, kw in (("default", dict()), ("explicit", dict(augment_intensity=0.0, augment_m=1, augment_k=1)),
                    ("shift", dict(augment_shift=4)), ("intensity", dict(augment_shift=4, augment_intensity=0.05)),
                    ("drq", DRQ)):
        names[tag] = update_graph(_agent(**kw), _memory(), tmp_path / f"{tag}.dot", monkeypatch)
    assert names["explicit"] == names["default"], "the defaults set explicitly leave the update graph as it is"
    assert "k_gather_aug" not in names["default"] and "k_c51_dueling_avg" not in names["default"]
    assert [("k_gather_shift" if k == "k_gather_aug" else k) for k in names["intensity"]] == names["shift"]
    assert names["intensity"].count("k_gather_aug") == names["shift"].count("k_gather_shift") >= 1
    drq = names["drq"]
    assert "k_c51_dueling_avg" in drq and "k_c51_dueling" not in drq
    # the project's kernels of the intensity graph with the loss kernel swapped and the head backward over M B = 64 rows
    # (k_head_bwd1_wgrad + k_head_bwd1_dx in place of k_head_bwd1: one launch more, DESIGN.md §3); cuDNN may pick other conv
    # kernels for the larger batch, so library kernels are not compared
    own = lambda ks: [k for k in ks if k.startswith("k_")]
    want = []
    for k in own(names["intensity"]):
        want += {"k_c51_dueling": ["k_c51_dueling_avg"], "k_head_bwd1": ["k_head_bwd1_wgrad", "k_head_bwd1_dx"]}.get(k, [k])
    assert own(drq) == want


def test_resume_equals_never_stopping(tmp_path):
    from test_gpu_checkpoint import _agent as ck_agent
    from test_gpu_checkpoint import _assert_same, _before_update, _fresh_memory, _state, _update
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
    assert (hp["augment_intensity"], hp["augment_m"], hp["augment_k"]) == (0.05, 2, 2)
    ag, mem = ck_agent(seed=77, **DRQ), _fresh_memory()
    ag.load_checkpoint(str(tmp_path / "ck"), mem)
    for step in range(save_at, total):
        if step > save_at:
            _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _assert_same(run_a, _state(ag, mem, losses))

    ck_agent(augment_intensity=0.0, augment_m=1, augment_k=1).save_checkpoint(str(tmp_path / "plain"))
    hp = json.load(open(tmp_path / "plain" / "rank0" / "manifest.json"))["hyper_parameters"]
    assert not {"augment_intensity", "augment_m", "augment_k"} & set(hp)


def test_learn_stats_hold_the_averaged_loss():
    ag = _agent(learn_stats=8, **DRQ)
    mem = _memory()
    for _ in range(3):
        ag.reset_noise()
        ag.learn(mem)
    torch.cuda.synchronize()
    rec = ag.learn_stats()
    assert len(rec["loss_mean"]) == 3
    assert rec["loss_mean"][-1] == pytest.approx(float(cpu(ag.last_loss).astype(np.float64).mean()), rel=1e-6)
    assert rec["loss_max"][-1] == cpu(ag.last_loss).max()
    m = cpu(ag._stats["last"]["m"]).astype(np.float64)
    assert rec["target_mean"][-1] == pytest.approx(float((m @ cpu(ag.support).astype(np.float64)).mean()), rel=1e-5)
    # q(s, a) of the taken action from copy 0's online rows (the first B rows of z), not copy 1's
    z, B, A, Z = ag._stats["last"]["z"].double(), ag.batch_size, ag.action_space, ag.atoms
    acts, sup = mem._last.actions, ag.support.double()

    def q_mean(rows):
        zr = z[rows]
        q = zr[:, :Z].unsqueeze(1) + zr[:, Z:].view(-1, A, Z) - zr[:, Z:].view(-1, A, Z).mean(1, keepdim=True)
        return float((torch.softmax(q[torch.arange(B, device=q.device), acts], 1) * sup).sum(1).mean())

    q0, q1 = q_mean(slice(0, B)), q_mean(slice(B, 2 * B))
    assert rec["q_mean"][-1] == pytest.approx(q0, rel=1e-5, abs=1e-6)
    assert abs(q1 - q0) > 1e-4, "the copies differ, so the check above sees which copy was used"


def test_acting_and_evaluation_are_not_augmented():
    kw = dict(architecture="data-efficient", hidden_size=64)
    aug, plain = _agent(**DRQ, **kw), _agent(**kw)
    val, _ = synthetic_ring(256, seed=4)
    states = val.iter_states(0, 8)
    for i in range(4):
        assert aug.act(states[i]) == plain.act(states[i])
    assert aug.evaluate_q_memory(val) == plain.evaluate_q_memory(val)


def test_refusals():
    from rainbow_b200 import RainbowB200Error
    kw = dict(architecture="data-efficient", hidden_size=64)
    for bad in (dict(augment_intensity=-0.01), dict(augment_intensity=0.51), dict(augment_intensity=float("nan")),
                dict(augment_m=0), dict(augment_k=9)):
        with pytest.raises(ValueError):
            _agent(**bad, **kw)
    ag = _agent(**DRQ, **kw)
    numpy_mem, _ = synthetic_ring(1024, seed=5, rng="numpy")
    with pytest.raises(ValueError):
        ag.learn(numpy_mem)
    with pytest.raises(ValueError):
        numpy_mem.sample(8, intensity=0.05)

    class Foreign:
        history = 4

        def sample(self, batch_size):
            raise AssertionError("not reached: the agent refuses first")

    with pytest.raises(RainbowB200Error):
        _agent(augment_intensity=0.05, **kw).learn(Foreign())
    for bad in (dict(fused_head=False, augment_m=2), dict(batch_size=512, augment_m=2)):
        refused, mem = _agent(cuda_graph=False, **bad, **kw), _memory()
        counter, tree = mem._rng_counter.clone(), mem.transitions.tree.clone()
        with pytest.raises(RainbowB200Error, match="fused head"):
            refused.learn(mem)
        assert torch.equal(mem._rng_counter, counter) and torch.equal(mem.transitions.tree, tree), "nothing sampled"
        assert int(refused.optimiser.step_count.item()) == 0
    assert int(ag.optimiser.step_count.item()) == 0, "a refused learn() does nothing"
    # intensity alone works on the library head: it lives in the gather
    lib_head = _agent(fused_head=False, cuda_graph=False, augment_intensity=0.05, **kw)
    lib_head.learn(_memory())
    assert torch.isfinite(lib_head.last_loss).all()
