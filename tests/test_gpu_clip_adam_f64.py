"""rb_clip_adam (global-norm clip + Adam on flat buffers: k_sqnorm, then k_clip_adam) through its C ABI against the float64
reference of tests/adam_ref.py, per element (|err| <= TAU * scale), one step at a time: every step starts from the kernel's
own state, so errors do not compound.  The cases cover
 * P of 1, 3, 4, 5 and 4097 (one CTA, partly idle; the scalar path whenever P % 4 != 0), around ADAM_MAX_CTAS * 256 * 4
   = 1 081 344 (where the vector loop's grid stride starts to wrap) and a 6.9 M-element buffer (the C2 model's, several
   rounds of the grid stride);
 * each of the four buffers offset by 1 to 3 floats (the scalar path at P % 4 == 0);
 * grad_scale 1, 0.5 and 1/8; a gradient norm below, above and within rounding of max_norm; zero, tiny (v' subnormal)
   and large gradients; step_count from 0, 9 and 10^6; betas (0.9, 0.999) and (0.5, 0.9); eps 1.5e-4 and 1e-8 (where
   sqrt(v') dominates the denominator and the approximate sqrt / reciprocal show most);
 * gate NULL, 1 and 0 (0: parameters, moments and step_count bitwise unchanged, the norm still written);
 * norm_out NULL (the same step bitwise), the completion ticket back to 0 after every call, and three graph replays of a
   captured step bitwise equal to three eager steps.
Observed largest |err| / scale per output go to $RB_PARITY_OBSERVED when that variable is set."""
import numpy as np
import pytest
import torch

import adam_ref as AR
import head_ref as R
from test_gpu_head_f64 import record
from test_gpu_parity import DEV

pytestmark = pytest.mark.gpu

VEC_WRAP = 1056 * 256 * 4          # ADAM_MAX_CTAS (8 per SM, 132 SMs) * ADAM_THREADS * 4 floats


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


def stream():
    return torch.cuda.current_stream().cuda_stream


# (P, buffer offsets (p, g, m, v) in floats, grad_scale, clip, gradient, step_count, betas, eps, gate, lr)
CASES = [
    (1, (0, 0, 0, 0), 1.0, "below", "normal", 0, (0.9, 0.999), 1.5e-4, None, 1e-3),
    (3, (0, 0, 0, 0), 1.0, "above", "normal", 9, (0.9, 0.999), 1e-8, None, 6.25e-5),
    (4, (0, 0, 0, 0), 0.5, "at", "normal", 0, (0.9, 0.999), 1.5e-4, 1, 1e-3),
    (5, (0, 0, 0, 0), 0.5, "below", "normal", 10 ** 6, (0.5, 0.9), 1e-8, None, 1e-3),
    (4097, (0, 0, 0, 0), 0.125, "above", "normal", 9, (0.9, 0.999), 1.5e-4, None, 6.25e-5),
    (VEC_WRAP - 4, (0, 0, 0, 0), 1.0, "above", "normal", 9, (0.9, 0.999), 1e-8, None, 1e-3),
    (VEC_WRAP, (0, 0, 0, 0), 0.5, "below", "normal", 0, (0.9, 0.999), 1.5e-4, 1, 6.25e-5),
    (VEC_WRAP + 4, (0, 0, 0, 0), 0.125, "at", "normal", 10 ** 6, (0.5, 0.9), 1e-8, None, 1e-3),
    (VEC_WRAP + 3, (0, 0, 0, 0), 1.0, "above", "normal", 0, (0.9, 0.999), 1.5e-4, None, 1e-3),
    (6_875_136, (0, 0, 0, 0), 1.0, "above", "normal", 9, (0.9, 0.999), 1.5e-4, None, 6.25e-5),
    (4096, (1, 0, 0, 0), 1.0, "above", "normal", 9, (0.9, 0.999), 1e-8, None, 1e-3),
    (4096, (0, 2, 0, 0), 0.5, "below", "normal", 0, (0.5, 0.9), 1.5e-4, None, 1e-3),
    (4096, (0, 0, 3, 0), 0.125, "at", "normal", 9, (0.9, 0.999), 1.5e-4, 1, 1e-3),
    (4096, (0, 0, 0, 1), 1.0, "above", "normal", 10 ** 6, (0.9, 0.999), 1e-8, None, 6.25e-5),
    (VEC_WRAP + 4, (0, 0, 0, 3), 1.0, "above", "normal", 9, (0.9, 0.999), 1.5e-4, None, 1e-3),
    (4096, (0, 0, 0, 0), 1.0, "below", "zero", 9, (0.9, 0.999), 1.5e-4, None, 1e-3),
    (4096, (0, 0, 0, 0), 1.0, "below", "tiny", 0, (0.9, 0.999), 1e-8, None, 1e-3),
    (4099, (0, 0, 0, 0), 0.5, "below", "tiny", 9, (0.5, 0.9), 1.5e-4, None, 1e-3),
    (4100, (0, 0, 0, 0), 1.0, "below", "large", 9, (0.9, 0.999), 1e-8, None, 1e-3),
    (4100, (0, 0, 0, 0), 0.125, "above", "large", 0, (0.9, 0.999), 1.5e-4, 1, 1e-3),
    (4096, (0, 0, 0, 0), 1.0, "above", "normal", 9, (0.9, 0.999), 1.5e-4, 0, 1e-3),
    (5, (0, 0, 0, 0), 0.5, "below", "normal", 0, (0.9, 0.999), 1e-8, 0, 1e-3),
    (VEC_WRAP + 4, (0, 0, 0, 0), 1.0, "above", "normal", 10 ** 6, (0.5, 0.9), 1e-8, 0, 1e-3),
]


def _id(c):
    P, offs, gs, clip, gk, step, (b1, b2), eps, gate, lr = c
    return (f"P{P}" + ("-off" + "".join(map(str, offs)) if any(offs) else "") + f"-s{gs:g}-{clip}-{gk}-t{step}-b{b1:g}_{b2:g}"
            f"-eps{eps:g}-gate{gate}")


def _grad(P, kind, gen):
    if kind == "zero":
        return torch.zeros(P, device=DEV)
    g = torch.randn(P, device=DEV, generator=gen)
    if kind == "tiny":                                      # |g| in [1e-22, 1e-18]: (1 - b2) g^2 subnormal
        return g.sign() * torch.exp(torch.empty(P, device=DEV).uniform_(-50.7, -41.4, generator=gen))
    return g * (1e4 if kind == "large" else 1.0)


def _max_norm(gnorm, clip):
    """below: coef = 1 (10 at least: with the 1e-6 of clip_grad_norm_ a tiny norm would still clip); at: the fp32 norm,
    coef within rounding of 1 (the "at" gradients are scaled to norm 1000, so 1e-6 / norm is below fp32's resolution)."""
    return {"below": max(10 * gnorm, 10.0), "above": 0.1 * gnorm, "at": float(np.float32(gnorm))}[clip]


def _buffers(P, offs):
    """Four flat fp32 buffers of P elements, each starting `off` floats into a 16-byte aligned allocation."""
    return [torch.full((P + 3,), float("nan"), device=DEV)[o:o + P] for o in offs]


def _call(p, g, m, v, P, gs, max_norm, lr, b1, b2, eps, step, part, norm, gate):
    from rainbow_b200 import _lib
    L = lib()
    _lib.check(L.rb_clip_adam(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), P, gs, max_norm, lr, b1, b2, eps,
                              step.data_ptr(), part.data_ptr(), None if norm is None else norm.data_ptr(),
                              None if gate is None else gate.data_ptr(), stream()))


@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_clip_adam_f64(case):
    P, offs, gs, clip, gkind, step0, (b1, b2), eps, gate_v, lr = case
    seed = CASES.index(case)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    p, g, m, v = _buffers(P, offs)
    p.copy_(torch.randn(P, device=DEV, generator=gen) * 0.01)
    p[::7] = 0.0                                            # the update alone decides these
    gmag = {"zero": 0.0, "tiny": 1e-20, "large": 1e4, "normal": 1.0}[gkind] * gs
    if step0 == 0:
        m.zero_(), v.zero_()
    else:                                                   # moments of the gradient's size (after clipping)
        shrink = 0.1 if clip == "above" else 1.0
        m.copy_(torch.randn(P, device=DEV, generator=gen) * 0.3 * gmag * shrink)
        v.copy_(torch.rand(P, device=DEV, generator=gen).add_(0.5) * (gmag * shrink) ** 2)
    step = torch.full((1,), step0, dtype=torch.int64, device=DEV)
    part = torch.zeros(lib().rb_clip_adam_scratch_elems(), dtype=torch.float64, device=DEV)
    norm = torch.full((1,), float("nan"), device=DEV)
    gate = None if gate_v is None else torch.full((1,), gate_v, dtype=torch.int32, device=DEV)
    for it in range(2):
        g.copy_(_grad(P, gkind, gen))
        if clip == "at":
            g.mul_(1000.0 / float(g.double().mul(float(np.float32(gs))).norm()))
        ref_norm = float(g.double().mul(float(np.float32(gs))).norm())
        max_norm = _max_norm(ref_norm, clip)
        p0, m0, v0, t0 = p.clone(), m.clone(), v.clone(), int(step.item())
        if it == 0:                                         # norm_out NULL: the same step, bitwise
            _call(p, g, m, v, P, gs, max_norm, lr, b1, b2, eps, step, part, None, gate)
            p1, m1, v1 = p.clone(), m.clone(), v.clone()
            p.copy_(p0), m.copy_(m0), v.copy_(v0), step.fill_(t0)
        norm.fill_(float("nan"))
        _call(p, g, m, v, P, gs, max_norm, lr, b1, b2, eps, step, part, norm, gate)
        torch.cuda.synchronize()
        assert int(part.view(torch.int64)[-1]) == 0, "the completion ticket is back to 0"
        if it == 0:
            assert torch.equal(p, p1) and torch.equal(m, m1) and torch.equal(v, v1), "norm_out NULL changes the step"
        ref = AR.clip_adam(p0, g, m0, v0, t0, gs, max_norm, lr, b1, b2, eps)
        record("clip_adam.norm", R.assert_within("norm", norm, torch.tensor([ref["norm"][0]], dtype=torch.float64, device=DEV),
                                                 torch.tensor([ref["norm"][1]], dtype=torch.float64, device=DEV), AR.TAU))
        if gate_v == 0:                                     # a rejected batch: nothing moves but the norm
            assert torch.equal(p, p0) and torch.equal(m, m0) and torch.equal(v, v0), "gate 0 left the state alone"
            assert int(step.item()) == t0, "gate 0 does not advance step_count"
            continue
        assert int(step.item()) == t0 + 1
        for name, got in (("m", m), ("v", v), ("p", p)):
            val, scale = ref[name]
            record(f"clip_adam.{name}", R.assert_within(name, got, val, scale, AR.TAU))


def test_clip_adam_graph_replay_equals_eager():
    """Three replays of one captured step (the step count is read on the device each time) == three eager steps."""
    P = VEC_WRAP + 4
    gen = torch.Generator(device=DEV).manual_seed(3)
    state0 = [torch.randn(P, device=DEV, generator=gen) * 0.01, torch.zeros(P, device=DEV), torch.zeros(P, device=DEV)]
    g = torch.randn(P, device=DEV, generator=gen)
    args = (P, 1.0, 100.0, 1e-3, 0.9, 0.999, 1e-8)
    runs = []
    for graphed in (False, True):
        p, m, v = (t.clone() for t in state0)
        step = torch.zeros(1, dtype=torch.int64, device=DEV)
        part = torch.zeros(lib().rb_clip_adam_scratch_elems(), dtype=torch.float64, device=DEV)
        norm = torch.zeros(1, device=DEV)
        fn = lambda: _call(p, g, m, v, *args, step, part, norm, None)
        if graphed:
            graph = torch.cuda.CUDAGraph()
            torch.cuda.synchronize()
            with torch.cuda.graph(graph):
                fn()
            for _ in range(3):
                graph.replay()
        else:
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        assert int(step.item()) == 3 and int(part.view(torch.int64)[-1]) == 0
        runs.append((p, m, v, norm))
    for a, b in zip(*runs):
        assert torch.equal(a, b)
