"""Clip + AdamW with Adam state per parameter group without a GPU: tests/adamw_ref.py against torch's own
clip_grad_norm_ + AdamW, its bound TAU against an fp32 model of k_clip_adamw (5x above) and against the slips it must catch
(5x below), every refusal of rb_clip_adamw and rb_peer_adamw_gather (answered before any launch), the rb_adam_group
layout, the Agent's option checks and the checkpoint's group-count check."""
import argparse
import ctypes as C

import numpy as np
import pytest
import torch

import adam_ref as AR
import adamw_ref as AW
from test_c51_adam_bounds import APPROX, SLIP_MARGIN, _adam_state, _ratio, kernel_model

RB_ERR_INVAL, RB_ERR_RANGE = -22, -34
ONE = 4096   # a pointer that is never dereferenced: validation fails first
F32 = lambda x: float(np.float32(x))


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


# ---- the reference against torch ----------------------------------------------------------------------------------------
def test_adamw_ref_is_torch_clip_and_adamw_in_float64():
    """Six steps of two parameter groups (lambda 0.1 and 0.01) through clip_grad_norm_ over both and torch.optim.AdamW;
    before step 3 the second group's state is re-created (a restart), so from there its count runs behind the first's."""
    lr, b1, b2, eps = F32(1e-3), F32(0.9), F32(0.999), F32(1.5e-4)
    wds = (F32(0.1), F32(0.01))
    rs = np.random.RandomState(0)
    sizes = (96, 40)
    ws = [torch.nn.Parameter(torch.from_numpy((rs.standard_normal(n) * 0.1).astype(np.float32)).double()) for n in sizes]
    opt = torch.optim.AdamW([dict(params=[ws[0]], weight_decay=wds[0]), dict(params=[ws[1]], weight_decay=wds[1])],
                            lr=lr, betas=(b1, b2), eps=eps)
    P = sum(sizes)
    groups = [(0, sizes[0], wds[0]), (sizes[0], P, wds[1])]
    p = torch.cat([w.detach() for w in ws]).float()
    m, v = torch.zeros(P), torch.zeros(P)
    counts = [0, 0]
    for step in range(6):
        if step == 3:
            opt.state.pop(ws[1])
            m[sizes[0]:], v[sizes[0]:], counts[1] = 0.0, 0.0, 0
        g = torch.from_numpy(rs.standard_normal(P).astype(np.float32))
        max_norm = F32(0.5 * float(g.double().norm()))
        ref = AW.clip_adamw(p, g, m, v, groups, counts, 1.0, max_norm, lr, b1, b2, eps)
        ws[0].grad, ws[1].grad = g[:sizes[0]].double().clone(), g[sizes[0]:].double().clone()
        norm = torch.nn.utils.clip_grad_norm_(ws, max_norm)
        opt.step()
        assert abs(float(norm) - ref["norm"][0]) <= 1e-13 * ref["norm"][0]
        got_p = torch.cat([w.detach() for w in ws])
        got_m = torch.cat([opt.state[w]["exp_avg"] for w in ws])
        got_v = torch.cat([opt.state[w]["exp_avg_sq"] for w in ws])
        for name, got in (("p", got_p), ("m", got_m), ("v", got_v)):
            torch.testing.assert_close(got, ref[name][0], rtol=1e-12, atol=1e-300)
        assert [int(opt.state[w]["step"]) for w in ws] == [c + 1 for c in counts]
        # the next step starts from torch's state rounded to fp32, as the kernel would hold it, on both sides
        p, m, v = got_p.float(), got_m.float(), got_v.float()
        with torch.no_grad():
            for w in ws:
                st = opt.state[w]
                for t in (w, st["exp_avg"], st["exp_avg_sq"]):
                    t.copy_(t.float().double())
        counts = [c + 1 for c in counts]


# ---- the bound -----------------------------------------------------------------------------------------------------------
SETTINGS = [  # (group counts, grad_scale, clip factor, betas, eps, lr, lambdas)
    ((0, 9), 1.0, 0.1, (0.9, 0.999), 1.5e-4, 1e-4, (0.1, 0.01)),
    ((9, 0), 0.5, 10.0, (0.9, 0.999), 1e-8, 1e-3, (0.01, 0.1)),
    ((10 ** 6, 9), 0.125, 1.0, (0.5, 0.9), 1e-8, 1e-3, (0.1, 0.0)),
    ((9, 10 ** 6), 1.0, 0.5, (0.9, 0.999), 1.5e-4, 1e-4, (0.0, 0.1))]


def _state(P, counts, seed):
    p, g, m, v = _adam_state(P, 1, seed)
    h = P // 2
    p[:] = (np.random.RandomState(seed + 100).standard_normal(P)).astype(np.float32)   # |p| ~ 1: the decay shows
    p[::7] = 0.0                                       # the update alone decides these: where decay-order slips show
    for (b, e), t in zip(((0, h), (h, P)), counts):
        if t == 0:
            m[b:e], v[b:e] = 0.0, 0.0
    return p, g, m, v, [(0, h), (h, P)]


def kernel_model_w(p, g, m, v, ranges, counts, wds, gs, max_norm, lr, b1, b2, eps, sqrt_err=0.0, rcp_err=0.0, slip=None):
    """k_sqnorm + k_clip_adamw in numpy: per group, p = fl32(p d_g) with d_g = fl32(1 - lr lambda_g), then k_clip_adam's
    arithmetic (test_c51_adam_bounds.kernel_model) with the group's count.  The norm and clip are over all elements: the
    model feeds each group its gradient and the global max_norm scaled to give the global coefficient.  `slip` replaces one
    piece of the semantics by a mistake the bound must catch."""
    f = np.float32
    gsum = float(np.sum((g * f(gs)).astype(np.float32).astype(np.float64) ** 2))
    outs = [np.empty_like(p) for _ in range(3)]
    for gi, ((b, e), t, wd) in enumerate(zip(ranges, counts, wds)):
        d = f(1.0 - float(f(lr)) * float(f(wd)))
        if slip == "decay_without_lr":
            d = f(1.0 - float(f(wd)))
        if slip == "other_group_count":
            t = counts[1 - gi]
        pg, gg = p[b:e], g[b:e]
        if slip == "l2_in_gradient":          # torch.optim.Adam(weight_decay=): g + lambda p, no decoupled decay
            gg = (gg + f(wd) * pg / f(gs)).astype(np.float32)
        elif slip != "decay_after_step":
            pg = (pg * d).astype(np.float32)
        # k_clip_adam's clip of this group's part with the global norm: the model computes the norm of what it is given,
        # so pass a max_norm that yields the global coefficient for this group's own norm
        gnorm = float(np.sqrt(np.sum((gg * f(gs)).astype(np.float32).astype(np.float64) ** 2)))
        coef = min(max_norm / (np.sqrt(gsum) + 1e-6), 1.0)
        mn = coef * (gnorm + 1e-6) if coef < 1.0 else 1e30
        p1, m1, v1, _ = kernel_model(pg, gg, m[b:e], v[b:e], t, gs, mn, lr, b1, b2, eps, sqrt_err, rcp_err)
        if slip == "decay_after_step":
            p1 = (p1 * d).astype(np.float32)
        outs[0][b:e], outs[1][b:e], outs[2][b:e] = p1, m1, v1
    return outs


def test_adamw_bound_is_5x_above_fp32_arithmetic():
    worst = {}
    for i, (counts, gs, clipf, (b1, b2), eps, lr, wds) in enumerate(SETTINGS):
        p, g, m, v, ranges = _state(4096, counts, 20 + i)
        max_norm = clipf * float(np.linalg.norm(g.astype(np.float64) * F32(gs)))
        ref = AW.clip_adamw(*(torch.from_numpy(x) for x in (p, g, m, v)), [(b, e, w) for (b, e), w in zip(ranges, wds)],
                            counts, gs, max_norm, lr, b1, b2, eps)
        for se in (-APPROX, 0.0, APPROX):
            for re in (-APPROX, 0.0, APPROX):
                res = kernel_model_w(p, g, m, v, ranges, counts, wds, gs, max_norm, lr, b1, b2, eps, se, re)
                for k, x in zip(("p", "m", "v"), res):
                    worst[k] = max(worst.get(k, 0.0), _ratio(torch.from_numpy(x), *ref[k]))
    for k, r in worst.items():
        assert SLIP_MARGIN * r <= AW.TAU, (k, worst)


@pytest.mark.parametrize("slip", ["decay_after_step", "decay_without_lr", "l2_in_gradient", "other_group_count"])
def test_adamw_slips_are_5x_above_tau(slip):
    counts, gs, (b1, b2), eps, lr, wds = (0, 10 ** 6), 1.0, (0.9, 0.999), 1.5e-4, 1e-3, (0.1, 0.1)
    if slip == "other_group_count":
        counts = (1, 9)
    p, g, m, v, ranges = _state(4096, counts, 7)
    max_norm = 10.0 * float(np.linalg.norm(g.astype(np.float64)))
    ref = AW.clip_adamw(*(torch.from_numpy(x) for x in (p, g, m, v)), [(b, e, w) for (b, e), w in zip(ranges, wds)],
                        counts, gs, max_norm, lr, b1, b2, eps)
    p1 = kernel_model_w(p, g, m, v, ranges, counts, wds, gs, max_norm, lr, b1, b2, eps, slip=slip)[0]
    worst = _ratio(torch.from_numpy(p1), *ref["p"])
    assert worst >= SLIP_MARGIN * AW.TAU, (slip, worst)


def test_adamw_ref_equals_adam_ref_without_decay():
    p, g, m, v = (torch.from_numpy(x) for x in _adam_state(1000, 9, 5))
    a = AR.clip_adam(p, g, m, v, 9, 0.5, 3.0, 1e-3, 0.9, 0.999, 1e-8)
    w = AW.clip_adamw(p, g, m, v, [(0, 400, 0.0), (400, 1000, 0.0)], [9, 9], 0.5, 3.0, 1e-3, 0.9, 0.999, 1e-8)
    for k in ("p", "m", "v"):
        torch.testing.assert_close(w[k][0], a[k][0], rtol=1e-15, atol=0)


# ---- the C ABI -----------------------------------------------------------------------------------------------------------
def groups(*rows):
    from rainbow_b200 import _lib
    return (_lib.AdamGroup * max(1, len(rows)))(*[_lib.AdamGroup(*r) for r in rows])


def test_adam_group_layout_and_signatures():
    from rainbow_b200 import _lib
    # rb_adam_group: int64 begin, end; float weight_decay (24 bytes with the trailing padding)
    assert C.sizeof(_lib.AdamGroup) == 24 and _lib.AdamGroup.end.offset == 8 and _lib.AdamGroup.weight_decay.offset == 16
    assert _lib.MAX_ADAM_GROUPS == 4
    assert len(_lib.SIGNATURES["rb_clip_adamw"][1]) == 19 and len(_lib.SIGNATURES["rb_peer_adamw_gather"][1]) == 24
    assert _lib.ALL_KERNEL_IDS[-2:] == ["target_ema", "param_reset"], "no new profiling id"


def test_clip_adamw_refusals_without_gpu():
    L = lib()
    good = [(0, 64, 0.1), (64, 100, 0.0)]

    def call(rows, P=100, n=None, lr=1e-3, ptrs=None):
        q = ptrs or dict(param=ONE, grad=ONE, m=ONE, v=ONE, groups=groups(*rows), step=ONE, gsteps=ONE, part=ONE)
        return L.rb_clip_adamw(q["param"], q["grad"], q["m"], q["v"], P, 1.0, 10.0, lr, 0.9, 0.999, 1e-8, q["groups"],
                               len(rows) if n is None else n, q["step"], q["gsteps"], q["part"], None, None, None)

    base = dict(param=ONE, grad=ONE, m=ONE, v=ONE, groups=groups(*good), step=ONE, gsteps=ONE, part=ONE)
    for k in base:
        assert call(good, ptrs=dict(base, **{k: None})) == RB_ERR_INVAL, k
        assert b"null" in L.rb_last_error()
    assert call(good, P=0) == RB_ERR_INVAL
    for n in (0, -1, 5):
        assert call(good, n=n) == RB_ERR_RANGE, n
    assert call([(0, 20, 0.0), (20, 40, 0.0), (40, 60, 0.0), (60, 80, 0.0), (80, 100, 0.0)]) == RB_ERR_RANGE
    bad_tables = [
        [(4, 64, 0.1), (64, 100, 0.0)],            # a gap before the first group
        [(0, 60, 0.1), (64, 100, 0.0)],            # a gap between groups
        [(0, 68, 0.1), (64, 100, 0.0)],            # an overlap
        [(64, 100, 0.0), (0, 64, 0.1)],            # unsorted
        [(0, 64, 0.1), (64, 64, 0.0), (64, 100, 0.0)],   # an empty group
        [(0, 64, 0.1), (64, 96, 0.0)],             # the last group ends before P
        [(0, 64, 0.1), (64, 104, 0.0)],            # ... or after it
    ]
    for rows in bad_tables:
        assert call(rows) == RB_ERR_RANGE, rows
        assert b"tile" in L.rb_last_error()
    assert call([(0, 62, 0.1), (62, 100, 0.0)]) == RB_ERR_RANGE        # a begin that is not a multiple of 4
    assert b"multiple of 4" in L.rb_last_error()
    for wd in (-0.1, -1e-30, float("nan"), float("inf")):
        assert call([(0, 64, 0.1), (64, 100, wd)]) == RB_ERR_RANGE, wd
        assert b"weight_decay" in L.rb_last_error()
    # fl32(lr) fl32(lambda) >= 1: the decay factor would be <= 0
    assert call([(0, 100, 1.0)], lr=1.0) == RB_ERR_RANGE
    assert call([(0, 100, 2000.0)], lr=1e-3) == RB_ERR_RANGE
    assert call([(0, 100, F32(1.0 / F32(0.3)) * 1.000001)], lr=0.3) == RB_ERR_RANGE


def test_peer_adamw_gather_refusals_without_gpu():
    L = lib()
    arr = lambda t, *v: (t * len(v))(*v)
    one = arr(C.c_void_p, ONE)
    begin, length = arr(C.c_int64, 0), arr(C.c_int64, 64)

    def call(wd=(0.1,), steps=ONE, lr=1e-3, n_seg=1, wd_arr="given"):
        w = arr(C.c_float, *wd) if wd_arr == "given" else None
        return L.rb_peer_adamw_gather(one, one, one, 1, 0, n_seg, begin, length, w, ONE, ONE, ONE, 10.0, lr, 0.9, 0.999,
                                      1e-8, ONE, steps, ONE, ONE, None, None, None)

    assert call(wd_arr=None) == RB_ERR_INVAL and b"null" in L.rb_last_error()
    assert call(steps=None) == RB_ERR_INVAL and b"null" in L.rb_last_error()
    assert call(n_seg=3) == RB_ERR_RANGE
    for wd in (-0.1, float("nan"), float("inf")):
        assert call(wd=(wd,)) == RB_ERR_RANGE and b"weight_decay" in L.rb_last_error()
    assert call(wd=(1.0,), lr=1.0) == RB_ERR_RANGE


# ---- Agent options and checkpoint scalars --------------------------------------------------------------------------------
def test_agent_option_checks():
    from rainbow_b200.agent import optimizer_options
    ns = argparse.Namespace
    assert optimizer_options(ns(learning_rate=1e-4)) == (0.0, False)
    assert optimizer_options(ns(learning_rate=1e-4, weight_decay=None, reset_optimizer=None)) == (0.0, False)
    assert optimizer_options(ns(learning_rate=1e-4, weight_decay=0.1, reset_optimizer=True)) == (0.1, True)
    assert optimizer_options(ns(learning_rate=0.5, weight_decay=1.9)) == (1.9, False)
    for bad in (dict(weight_decay=-0.1), dict(weight_decay=float("nan")), dict(weight_decay=float("inf")),
                dict(weight_decay=1e5), dict(learning_rate=1.0, weight_decay=1.0), dict(reset_optimizer=1),
                dict(reset_optimizer="yes")):
        with pytest.raises(ValueError):
            optimizer_options(ns(**dict(dict(learning_rate=1e-4), **bad)))


def test_group_optimiser_state_on_the_host_net():
    """FusedClipAdam's groups (encoder [0, conv_end), head [conv_end, numel)) and restart on a CPU-built net."""
    from rainbow_b200.agent import ENCODER, HEAD, FusedClipAdam
    from rainbow_b200.model import DQN
    torch.manual_seed(0)
    net = DQN(argparse.Namespace(atoms=51, hidden_size=256, architecture="data-efficient", history_length=4,
                                 noisy_std=0.1), 6)
    plain = FusedClipAdam(net, lr=1e-4, eps=1e-4, max_norm=10.0)
    assert not plain.grouped and not hasattr(plain, "group_steps")
    net = DQN(argparse.Namespace(atoms=51, hidden_size=256, architecture="data-efficient", history_length=4,
                                 noisy_std=0.1), 6)
    opt = FusedClipAdam(net, lr=1e-4, eps=1e-4, max_norm=10.0, weight_decay=0.1)
    assert opt.grouped and opt.groups == [(0, opt.conv_end), (opt.conv_end, opt.numel)] and opt.conv_end % 4 == 0
    assert [(g.begin, g.end, g.weight_decay) for g in opt._groups_c] == [(0, opt.conv_end, F32(0.1)),
                                                                       (opt.conv_end, opt.numel, F32(0.1))]
    opt.exp_avg.fill_(1.0), opt.exp_avg_sq.fill_(2.0)
    opt.set_group_step_counts([7, 5])
    assert opt.group_step_counts() == [7, 5]
    opt.restart_group(HEAD)
    assert opt.group_step_counts() == [7, 0]
    assert (opt.exp_avg[opt.conv_end:] == 0).all() and (opt.exp_avg_sq[opt.conv_end:] == 0).all()
    assert (opt.exp_avg[:opt.conv_end] == 1).all() and (opt.exp_avg_sq[:opt.conv_end] == 2).all()
    opt.restart_group(ENCODER)
    assert opt.group_step_counts() == [0, 0] and (opt.exp_avg == 0).all()
    with pytest.raises(Exception, match="group optimiser"):
        plain.restart_group(HEAD)


def test_group_optimiser_state_under_the_peer_optimiser(monkeypatch):
    """FusedClipAdam over the peer optimiser's layout (a stand-in for PeerOptimizerState: rank 2 of 4, no symmetric
    memory): the moments are this rank's shards of segment 0 = head, then segment 1 = encoder, and group_steps is in
    segment order.  restart_group must zero exactly the shard of the group's own segment, and the counts must map to
    [encoder, head]; step() hands the device counts and lambda to the peer step."""
    import rainbow_b200.peer as peer_mod
    from rainbow_b200.agent import ENCODER, HEAD, FusedClipAdam
    from rainbow_b200.model import DQN

    class StubPeer:
        shard_slices = peer_mod.PeerOptimizerState.shard_slices

        def __init__(self, numel, device, segments=None, group=None):
            self.world, self.rank, self.numel = 4, 2, numel
            self.segments = [s for s in segments if s[1] > s[0]]
            self.parts = [(e - b) // self.world for b, e in self.segments]
            self.shard = sum(self.parts)
            self.flat_param, self.flat_grad = torch.zeros(numel), torch.zeros(numel)
            self.exp_avg, self.exp_avg_sq = torch.zeros(self.shard), torch.zeros(self.shard)
            self.step_count, self.grad_norm = torch.zeros(1, dtype=torch.int64), torch.zeros(1)
            self.calls = []

        def step(self, max_norm, lr, betas, eps, weight_decay=None, seg_steps=None):
            self.calls.append((weight_decay, seg_steps))

    monkeypatch.setattr(peer_mod, "PeerOptimizerState", StubPeer)
    torch.manual_seed(0)
    net = DQN(argparse.Namespace(atoms=51, hidden_size=256, architecture="data-efficient", history_length=4,
                                 noisy_std=0.1), 6)
    opt = FusedClipAdam(net, lr=1e-4, eps=1e-4, max_norm=10.0, peer=True, weight_decay=0.1)
    assert opt.grouped and opt.peer.segments == [(opt.conv_end, opt.numel), (0, opt.conv_end)]
    # this rank's shards, from the layout alone: head part of segment 0 first, then the encoder part of segment 1
    hp, ep = (opt.numel - opt.conv_end) // 4, opt.conv_end // 4
    assert opt.exp_avg.numel() == hp + ep and hp != ep
    m0 = torch.arange(1, hp + ep + 1, dtype=torch.float32)
    opt.exp_avg.copy_(m0), opt.exp_avg_sq.copy_(2 * m0)
    opt.set_group_step_counts([7, 5])
    assert opt.group_steps.tolist() == [5, 7], "group_steps is in segment order: head, encoder"
    assert opt.group_step_counts() == [7, 5]
    opt.restart_group(ENCODER)
    assert not opt.exp_avg[hp:].any() and not opt.exp_avg_sq[hp:].any(), "the encoder's shard is zeroed"
    assert torch.equal(opt.exp_avg[:hp], m0[:hp]) and torch.equal(opt.exp_avg_sq[:hp], 2 * m0[:hp]), "the head's is kept"
    assert opt.group_step_counts() == [0, 5] and opt.group_steps.tolist() == [5, 0]
    opt.restart_group(HEAD)
    assert not opt.exp_avg.any() and not opt.exp_avg_sq.any() and opt.group_step_counts() == [0, 0]
    opt.step()
    (wd, seg_steps), = opt.peer.calls
    assert wd == 0.1 and seg_steps is opt.group_steps


def test_checkpoint_group_steps_check():
    from rainbow_b200 import _lib
    from rainbow_b200.checkpoint import check_group_steps
    check_group_steps(dict(optimiser_step=12))                                  # absent: loads as [12, 12]
    for ok in ([0, 0], [12, 3], [12, 12], [0, 12]):
        check_group_steps(dict(optimiser_step=12, optimiser_group_steps=ok))
    for bad in ([13, 0], [0, 13], [-1, 0], [1], [1, 2, 3], (1, 2), [1.0, 2], [True, 2], "12", 12, [None, 1]):
        with pytest.raises(_lib.RainbowB200Error, match="optimiser_group_steps"):
            check_group_steps(dict(optimiser_step=12, optimiser_group_steps=bad))
