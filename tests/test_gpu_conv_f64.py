"""The conv body's backward against the float64 reference of tests/conv_ref.py, per element (|err| <= tau * scale):

* rb_conv_wgrad (k_conv_wgrad_first<KW> + k_conv_wgrad_reduce) on every variant it ships: KW 3, 4, 5 and 8; both
  architectures' layer 0 at batch 1 to 512 and at every history length the kernel accepts; one band (OH < 16) and a
  ragged last band; OC % 4 != 0; exactly 256 threads; IH != IW; g and x one float off 16-byte alignment (the scalar
  staging); fewer than 4 partials (empty quarters) and partial counts that are no multiple of 4 or 32.  Each case asserts
  the variants it names, that its sentinel outputs are overwritten and guard elements past them untouched, that a second
  launch, a launch without the bias output and a CUDA-graph replay are bitwise equal, and that the graph ran
  k_conv_wgrad_first<KW> and the reduce.  The outputs also equal conv_ref's numpy model of the kernels' fp32 arithmetic,
  bitwise, on a sample of elements.
* rb_bias_grad at the (C, HW) of every call the learner makes, 1 to 512 rows, B HW below, at and above 256 threads and
  with a ragged last pass, and from a misaligned pointer; equal to the numpy model of k_bias_grad bitwise.
* Refused shapes write nothing; DQN._own_wgrad_ok agrees with what rb_conv_wgrad accepts at history 1 to 8, and the
  update graph holds our layer-0 kernels exactly where it says so.
* DQN.conv_backward_into_grads (deterministic cuDNN, TF32 off): every layer's gradients against the float64 chain of the
  learner's own fp32 activations, weights and ReLU sides; the last layer's bias (k_bias_grad on g_last) within TAU_BIAS,
  everything cuDNN's fp32 dgrad / wgrad produce or feed within TAU_LIB.
Observed largest |err| / scale go to $RB_PARITY_OBSERVED when that variable is set."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest
import torch

import conv_ref as R
import head_ref as H
from test_gpu_augment import update_graph
from test_gpu_head_f64 import graph_kernels
from test_gpu_parity import DEV, FakeEnv, make_args, synthetic_ring

pytestmark = pytest.mark.gpu

NAN = float("nan")
GUARD = 5                 # elements past each output that must stay untouched


@pytest.fixture(autouse=True)
def exact_fp32_cudnn():
    flags = (torch.backends.cudnn.deterministic, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


def stream():
    return torch.cuda.current_stream().cuda_stream


def record(key, value):
    """Largest observed |err| / scale per output, merged into $RB_PARITY_OBSERVED."""
    path = os.environ.get("RB_PARITY_OBSERVED")
    if not path:
        return
    data = json.load(open(path)) if os.path.exists(path) else {}
    data.setdefault("conv_f64_tau_wgrad", R.TAU_WGRAD)
    data.setdefault("conv_f64_tau_bias", R.TAU_BIAS)
    data.setdefault("conv_f64_tau_lib", R.TAU_LIB)
    data[key] = max(float(value), data.get(key, 0.0))
    with open(path, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)


def _offset(t, off):
    """A copy of t whose data starts `off` floats into its storage (off = 1: 4 bytes past 16-byte alignment)."""
    buf = torch.empty(t.numel() + off, dtype=t.dtype, device=t.device)
    out = buf[off:].view(t.shape)
    out.copy_(t)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# rb_conv_wgrad
def wg_variants(B, IC, IH, IW, OC, K, S, off):
    """The variants of rb_conv_wgrad a shape takes.  Mirrors rb_conv_wgrad / k_conv_wgrad_first in csrc/rb_head.cu
    (conv_wgrad_band_rows, the cp.async condition, the float4 row loads, the thread count); update them together."""
    OH, OW = (IH - K) // S + 1, (IW - K) // S + 1
    RB, nb = R.bands_of(OH)
    n_part = B * nb
    v = {f"KW{K}", "cp.async" if (IW % 4 == 0 and OW % 4 == 0 and off == 0) else "scalar staging"}
    if K % 4 == 0 and S % 4 == 0 and IW % 4 == 0:
        v.add("float4 rows")
    if OH < 16:
        v.add("one band")
    if OH % RB:
        v.add("ragged band")
    if OC % 4:
        v.add("OC % 4 != 0")
    if IC * K * -(-OC // 4) == 256:
        v.add("256 threads")
    if n_part < 4:
        v.add("n_part < 4")
    if n_part % 4 and n_part % 32 and n_part >= 4:
        v.add("n_part % 4, % 32 != 0")
    if IH != IW:
        v.add("IH != IW")
    if B == 512:
        v.add("512 rows")
    return v


def _wg_cases():
    cases = []   # (name, B, IC, IH, IW, OC, K, S, off, one_signed, names)
    for arch, hmax in (("canonical", 4), ("data-efficient", 6)):
        OC, K, S = R.ARCH[arch][0]
        for B in (1, 5, 32, 33, 64, 512):
            cases.append((f"{arch}-B{B}", B, 4, 84, 84, OC, K, S, 0, False, {f"KW{K}"} | ({"512 rows"} if B == 512 else set())))
        for h in range(1, hmax + 1):
            if h != 4:
                cases.append((f"{arch}-history{h}", 32, h, 84, 84, OC, K, S, 0, False, {f"KW{K}"}))
        cases.append((f"{arch}-B32-offset", 32, 4, 84, 84, OC, K, S, 1, False, {"scalar staging"}))
        cases.append((f"{arch}-B512-one-signed", 512, 4, 84, 84, OC, K, S, 0, True, {"512 rows"}))
    cases += [
        ("K4-S2-one-band", 7, 3, 30, 30, 16, 4, 2, 0, False, {"KW4", "one band"}),
        ("K3-S1-one-band", 2, 8, 13, 13, 24, 3, 1, 0, False, {"KW3", "one band", "n_part < 4"}),
        ("K3-OC7-B1", 1, 5, 20, 20, 7, 3, 2, 0, False, {"KW3", "OC % 4 != 0", "n_part < 4"}),
        ("K4-B3-one-band", 3, 3, 30, 30, 16, 4, 2, 0, False, {"KW4", "n_part < 4"}),
        ("OC30-256-threads", 9, 4, 84, 84, 30, 8, 4, 0, False, {"OC % 4 != 0", "256 threads", "ragged band"}),
        ("IH40-IW60", 9, 2, 40, 60, 20, 4, 2, 0, False, {"IH != IW", "scalar staging", "ragged band"}),
        ("IH84-IW100", 6, 4, 84, 100, 32, 8, 4, 0, False, {"IH != IW", "cp.async", "float4 rows"}),
        ("IH60-IW30-K5-S1", 4, 3, 60, 30, 13, 5, 1, 0, False, {"IH != IW", "KW5", "OC % 4 != 0"}),
    ]
    return cases


WG_CASES = _wg_cases()
REQUIRED = {"KW3", "KW4", "KW5", "KW8", "cp.async", "scalar staging", "float4 rows", "one band", "ragged band",
            "OC % 4 != 0", "256 threads", "n_part < 4", "n_part % 4, % 32 != 0", "IH != IW", "512 rows"}


def test_wgrad_cases_reach_every_variant():
    """Every case reaches the variants it names; together they reach every variant of REQUIRED, both architectures' layer 0
    at batch 1, 5, 32, 33, 64 and 512, every history length the kernel accepts, and the canonical shape misaligned."""
    reached = set()
    for name, B, IC, IH, IW, OC, K, S, off, _, names in WG_CASES:
        v = wg_variants(B, IC, IH, IW, OC, K, S, off)
        assert names <= v, (name, names - v)
        reached |= v
    assert REQUIRED <= reached, REQUIRED - reached
    for arch, hmax in (("canonical", 4), ("data-efficient", 6)):
        OC, K, S = R.ARCH[arch][0]
        shapes = {(c[1], c[2]) for c in WG_CASES if c[3:8] == (84, 84, OC, K, S) and not c[8]}
        assert {(B, 4) for B in (1, 5, 32, 33, 64, 512)} <= shapes
        assert {(32, h) for h in range(1, hmax + 1)} <= shapes
        assert IC_limit(OC, K) == hmax
    assert any(c[8] for c in WG_CASES if c[3:8] == (84, 84) + R.ARCH["canonical"][0])


def IC_limit(OC, K):
    """The largest input channel count (history length) rb_conv_wgrad takes at (OC, K): IC K ceil(OC / 4) <= 256."""
    return 256 // (K * -(-OC // 4))


def _wg_inputs(B, IC, IH, IW, OC, K, S, off, one_signed, seed):
    g_ = torch.Generator(device=DEV).manual_seed(seed)
    OH, OW = (IH - K) // S + 1, (IW - K) // S + 1
    x = torch.randint(0, 256, (B, IC, IH, IW), device=DEV, generator=g_).float() / 255
    g = torch.randn(B, OC, OH, OW, device=DEV, generator=g_) * (torch.rand(B, OC, OH, OW, device=DEV, generator=g_) > 0.5)
    g = (g.abs() if one_signed else g) * 1e-3
    return _offset(g, off), _offset(x, off)


class WGrad:
    def __init__(self, B, IC, IH, IW, OC, K, S):
        self.shape = (B, IC, IH, IW, OC, K, S)
        self.n_w = OC * IC * K * K
        n = lib().rb_conv_wgrad_scratch_elems(B, IC, IH, OC, K, S)
        assert n > 0
        self.scratch = torch.full((n,), NAN, device=DEV)

    def outputs(self):
        OC = self.shape[4]
        return torch.full((self.n_w + GUARD,), NAN, device=DEV), torch.full((OC + GUARD,), NAN, device=DEV)

    def __call__(self, g, x, out, bias):
        B, IC, IH, IW, OC, K, S = self.shape
        rc = lib().rb_conv_wgrad(g.data_ptr(), x.data_ptr(), B, IC, IH, IW, OC, K, S, self.scratch.data_ptr(), out.data_ptr(),
                                 None if bias is None else bias.data_ptr(), stream())
        assert rc == 0, lib().rb_last_error()


_WG_KERNEL = re.compile(r"k_conv_wgrad_first(?:<\s*(\d+)\s*>|ILi(\d+)E)")


@pytest.mark.parametrize("case", WG_CASES, ids=[c[0] for c in WG_CASES])
def test_conv_wgrad_f64(case, tmp_path):
    name, B, IC, IH, IW, OC, K, S, off, one_signed, _ = case
    g, x = _wg_inputs(B, IC, IH, IW, OC, K, S, off, one_signed, seed=B * 131 + IC * 17 + OC + K)
    run = WGrad(B, IC, IH, IW, OC, K, S)
    n_w = run.n_w
    out, bias = run.outputs()
    run(g, x, out, bias)
    torch.cuda.synchronize()
    assert torch.isnan(out[n_w:]).all() and torch.isnan(bias[OC:]).all(), "written past the last output"
    ref, scale = R.wgrad(g, x, K, S)
    bref, bscale = R.bias(g)
    record("wgrad.w", H.assert_within("weight gradient", out[:n_w].view(OC, IC, K, K), ref, scale, R.TAU_WGRAD))
    record("wgrad.b", H.assert_within("bias gradient", bias[:OC], bref, bscale, R.TAU_BIAS))

    out2, bias2 = run.outputs()
    run(g, x, out2, bias2)
    out3, _ = run.outputs()
    run(g, x, out3, None)                                              # bias_out = NULL
    out4, bias4 = run.outputs()
    graph, _, dot = graph_kernels(lambda: run(g, x, out4, bias4), tmp_path / "wgrad.dot")
    kw = {int(a or b) for a, b in _WG_KERNEL.findall(dot)}
    assert kw == {K} and "k_conv_wgrad_reduce" in dot, f"the graph ran k_conv_wgrad_first<{kw}>, expected <{K}> + reduce"
    for what, (o, b) in (("second launch", (out2, bias2)), ("graph replay", (out4, bias4))):
        assert torch.equal(o[:n_w], out[:n_w]) and torch.equal(b[:OC], bias[:OC]), f"{what}: bitwise equal"
    assert torch.equal(out3[:n_w], out[:n_w]), "the weights without a bias output equal those with one, bitwise"
    assert torch.isnan(out3[n_w:]).all()
    del graph


@pytest.mark.parametrize("case", WG_CASES, ids=[c[0] for c in WG_CASES])
def test_conv_wgrad_is_the_fp32_model(case):
    """The kernels compute what conv_ref's numpy model of their fp32 arithmetic computes, bitwise: on 24 sampled weight
    elements and every bias element."""
    name, B, IC, IH, IW, OC, K, S, off, one_signed, _ = case
    g, x = _wg_inputs(B, IC, IH, IW, OC, K, S, off, one_signed, seed=B * 131 + IC * 17 + OC + K)
    run = WGrad(B, IC, IH, IW, OC, K, S)
    out, bias = run.outputs()
    run(g, x, out, bias)
    elems = np.random.RandomState(B + K).choice(run.n_w, min(24, run.n_w), replace=False)
    w, b = R.wgrad_model(g.cpu().numpy(), x.cpu().numpy(), K, S, elems)
    got_w, got_b = out.cpu().numpy()[elems], bias.cpu().numpy()[:OC]
    assert np.array_equal(got_w.view(np.uint32), w.view(np.uint32)), (name, np.abs(got_w - w).max())
    assert np.array_equal(got_b.view(np.uint32), b.view(np.uint32)), (name, np.abs(got_b - b).max())


# ---------------------------------------------------------------------------------------------------------------------
# rb_bias_grad
def _bg_cases():
    cases = []   # (C, HW, rows, off)
    for C_, HW in R.BIAS_SHAPES:
        for rows in (1, 3, 33, 512):
            cases.append((C_, HW, rows, 0))
    cases += [(64, 9, 28, 0), (8, 16, 15, 0), (8, 16, 16, 0), (8, 16, 17, 0), (64, 81, 33, 1), (64, 49, 5, 1)]
    return cases


BG_CASES = _bg_cases()


def test_bias_grad_cases_reach_every_pass_shape():
    n = [rows * HW for _, HW, rows, _ in BG_CASES]
    assert any(v < 256 for v in n) and any(v == 256 for v in n) and any(v > 256 for v in n)
    assert any(v > 256 and v % 256 for v in n), "a ragged last pass"
    assert any(c[3] for c in BG_CASES), "a misaligned pointer"
    assert {(c[0], c[1]) for c in BG_CASES} >= set(R.BIAS_SHAPES)
    assert {c[2] for c in BG_CASES} >= {1, 512}


@pytest.mark.parametrize("case", BG_CASES, ids=[f"C{c[0]}-HW{c[1]}-rows{c[2]}" + ("-offset" if c[3] else "") for c in BG_CASES])
def test_bias_grad_f64(case):
    C_, HW, rows, off = case
    gen = torch.Generator(device=DEV).manual_seed(C_ * 1000 + HW + rows)
    g = torch.randn(rows, C_, HW, device=DEV, generator=gen) * (torch.rand(rows, C_, HW, device=DEV, generator=gen) > 0.5)
    g = _offset(g * 1e-3, off)
    L = lib()
    outs = []
    for _ in range(2):
        out = torch.full((C_ + GUARD,), NAN, device=DEV)
        assert L.rb_bias_grad(g.data_ptr(), rows, C_, HW, out.data_ptr(), stream()) == 0, L.rb_last_error()
        outs.append(out)
    torch.cuda.synchronize()
    out = outs[0]
    assert torch.isnan(out[C_:]).all(), "written past the last channel"
    record("bias_grad.b", H.assert_within("bias gradient", out[:C_], *R.bias(g), R.TAU_BIAS))
    assert torch.equal(outs[1][:C_], out[:C_]), "a second launch is bitwise equal"
    model = R.bias_grad_model(g.cpu().numpy())
    assert np.array_equal(out[:C_].cpu().numpy().view(np.uint32), model.view(np.uint32)), "equal to the fp32 model, bitwise"


# ---------------------------------------------------------------------------------------------------------------------
# refusals and dispatch
REFUSED = [   # (why, B, IC, IH, IW, OC, K, S)
    ("kernel size 7", 2, 4, 84, 84, 32, 7, 4),
    ("320 threads", 2, 5, 84, 84, 32, 8, 4),
    ("partials past 2^31 - 1 floats", 37304, 4, 84, 84, 32, 8, 4),
    ("slab past 200 KB of shared memory", 2, 2, 84, 8000, 32, 8, 4),
]


@pytest.mark.parametrize("case", REFUSED, ids=[c[0] for c in REFUSED])
def test_conv_wgrad_refusals_write_nothing(case):
    """Each refusal is RB_ERR_RANGE before any launch (the buffers are a few floats: nothing may read them)."""
    _, B, IC, IH, IW, OC, K, S = case
    small = torch.zeros(64, device=DEV)
    scratch = torch.full((64,), NAN, device=DEV)
    out = torch.full((64,), NAN, device=DEV)
    bias = torch.full((64,), NAN, device=DEV)
    L = lib()
    assert L.rb_conv_wgrad(small.data_ptr(), small.data_ptr(), B, IC, IH, IW, OC, K, S, scratch.data_ptr(), out.data_ptr(),
                           bias.data_ptr(), stream()) == -34
    torch.cuda.synchronize()
    assert torch.isnan(scratch).all() and torch.isnan(out).all() and torch.isnan(bias).all()


def _net(arch, history, seed=0):
    from rainbow_b200.model import DQN
    torch.manual_seed(seed)
    return DQN(make_args(architecture=arch, history_length=history, hidden_size=64), 6).to(DEV)


@pytest.mark.parametrize("arch", list(R.ARCH))
def test_own_wgrad_dispatch_agrees_with_the_kernel(arch):
    """DQN._own_wgrad_ok is true exactly where rb_conv_wgrad takes layer 0's shape (history 1 to 8, batch 2)."""
    L = lib()
    OC, K, S = R.ARCH[arch][0]
    OH = (84 - K) // S + 1
    took = []
    for h in range(1, 9):
        net = _net(arch, h)
        m = net.conv_layers()[0]
        m.weight.grad, m.bias.grad = torch.full_like(m.weight, NAN), torch.full_like(m.bias, NAN)
        a_in = torch.rand(2, h, 84, 84, device=DEV)
        g = torch.randn(2, OC, OH, OH, device=DEV)
        n = L.rb_conv_wgrad_scratch_elems(2, h, 84, OC, K, S)
        scratch = torch.empty(max(n, 1), device=DEV)
        rc = L.rb_conv_wgrad(g.data_ptr(), a_in.data_ptr(), 2, h, 84, 84, OC, K, S, scratch.data_ptr(), m.weight.grad.data_ptr(),
                             m.bias.grad.data_ptr(), stream())
        assert rc in (0, -34)
        assert net._own_wgrad_ok(m, a_in) == (rc == 0), (h, rc)
        took.append(rc == 0)
        torch.cuda.synchronize()
        if rc != 0:
            assert torch.isnan(m.weight.grad).all(), "a refused call writes nothing"
    assert took == [h <= IC_limit(OC, K) for h in range(1, 9)]


@pytest.mark.parametrize("arch,history", [("canonical", 4), ("canonical", 5), ("data-efficient", 6), ("data-efficient", 7)])
def test_update_graph_runs_our_layer0_kernels_where_dispatch_says(arch, history, tmp_path, monkeypatch):
    from rainbow_b200.agent import Agent
    torch.manual_seed(3)
    ag = Agent(make_args(architecture=arch, history_length=history, batch_size=32), FakeEnv(6))
    mem, _ = synthetic_ring(4096, seed=3, args=dict(history_length=history))
    names = update_graph(ag, mem, tmp_path / "update.dot", monkeypatch)
    dot = open(tmp_path / "update.dot").read()
    on = ag.online_net
    m = on.conv_layers()[0]
    own = on._own_wgrad_ok(m, torch.empty(32, history, 84, 84, device=DEV))
    assert own == (history <= IC_limit(*R.ARCH[arch][0][:2]))
    kw = {int(a or b) for a, b in _WG_KERNEL.findall(dot)}
    assert kw == ({R.ARCH[arch][0][1]} if own else set()), (kw, own)
    assert ("k_conv_wgrad_reduce" in names) == own


# ---------------------------------------------------------------------------------------------------------------------
# the chain
CHAIN_CASES = [(arch, 4, rows, False) for arch in R.ARCH for rows in (1, 32, 64, 512)] + \
              [(arch, 4, 32, True) for arch in R.ARCH] + \
              [("canonical", 5, 32, False), ("canonical", 5, 512, False), ("data-efficient", 7, 32, False)]


def _chain_id(c):
    arch, h, rows, drq = c
    return f"{arch}-history{h}-" + (f"drq-M2-B{rows}" if drq else f"rows{rows}")


@pytest.mark.parametrize("case", CHAIN_CASES, ids=[_chain_id(c) for c in CHAIN_CASES])
def test_conv_backward_chain_f64(case):
    """conv_backward_into_grads from a ReLU-masked g_last on the learner's own conv_forward_saving activations.  DrQ M = 2
    at batch 32: 64 rows, the second 32 a shifted copy of the first (the copies' gradients sum in the same kernels)."""
    arch, history, rows, drq = case
    net = _net(arch, history, seed=rows + history)
    gen = torch.Generator(device=DEV).manual_seed(rows * 7 + history)
    x = torch.randint(0, 256, (rows, history, 84, 84), device=DEV, generator=gen).float() / 255
    if drq:
        x = torch.cat([x, torch.roll(x, shifts=(3, -2), dims=(2, 3))])
    layers = net.conv_layers()
    with torch.no_grad():
        acts = net.conv_forward_saving(x)
        g_last = torch.randn(acts[-1].shape, device=DEV, generator=gen) * (acts[-1] > 0) * 1e-3

    def run():
        for m in layers:
            m.weight.grad, m.bias.grad = torch.full_like(m.weight, NAN), torch.full_like(m.bias, NAN)
        side = torch.cuda.Stream()
        done = net.conv_backward_into_grads(acts, g_last, side)
        torch.cuda.current_stream().wait_event(done)
        torch.cuda.synchronize()
        return [(m.weight.grad.clone(), m.bias.grad.clone()) for m in layers]

    got = run()
    assert net._own_wgrad_ok(layers[0], acts[0]) == (history <= IC_limit(*R.ARCH[arch][0][:2]))
    ref = R.chain(acts, [m.weight.detach() for m in layers], [m.stride[0] for m in layers], g_last)
    last = len(layers) - 1
    own0 = net._own_wgrad_ok(layers[0], acts[0])
    for li, (gw, gb) in enumerate(got):
        tau_b = R.TAU_BIAS if li == last else R.TAU_LIB                 # k_bias_grad on g_last itself / fed by cuDNN's dgrad
        if li == 0 and own0:                                            # k_conv_wgrad_first, fed by cuDNN's dgrad
            record("chain.layer0.w", H.assert_within("layer 0 weight", gw, *ref[li]["w"], R.TAU_LIB))
        else:                                                           # cuDNN's wgrad: normwise (conv_ref.wgrad_normwise)
            record(f"chain.layer{li}.w_cudnn_normwise",
                   H.assert_within(f"layer {li} weight (cuDNN)", gw, ref[li]["w"][0], ref[li]["wn"], R.TAU_LIB))
            record(f"chain.layer{li}.w_cudnn_elementwise", H.err_ratio(gw, *ref[li]["w"], R.TAU_LIB)[0])
        record(f"chain.layer{li}.b", H.assert_within(f"layer {li} bias", gb, *ref[li]["b"], tau_b))
    again = run()
    for (a, b), (c, d) in zip(got, again):
        assert torch.equal(a, c) and torch.equal(b, d), "deterministic: a second backward is bitwise equal"
