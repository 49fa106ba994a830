"""The fused noisy dueling head through its C ABI (rb_head_forward / rb_head_logits / rb_q_values / rb_head_backward) against
the float64 reference of tests/head_ref.py, per element (|err| <= TAU * scale; TAU_TC / TAU_TC_WGRAD for the tensor-core products), on
every kernel variant that ships:

 * layer 1 on the tensor cores (k_head_fc1_tc, then k_head_reduce1 iff the launch splits K) or on FFMA (k_head_fc<., 1>),
   including hidden sizes whose CTAs walk 13 and 25 k tiles (the 4-stage TMA ring wraps several times and the eps_in
   chunks past the 8 kept in registers are loaded per stage), conv_features 32 (no split: bias + ReLU in the kernel) and
   row counts up to FusedHead.MAX_ROWS;
 * layer 2 single-pass (k_head_fc2) or split-K with last-CTA tickets (k_head_fc<., 2>: hidden >= 768, or debug bit 3);
 * the backward at B <= 32 with and without the ReLU mask of x, noisy and eval, up to hidden 1024 and actions * atoms
   1062 (the dh kernel's eps_out fallback past its 8 prefetched factors).
Each case asserts which kernels ran (the nodes of the forward captured as a CUDA graph), that every output was overwritten (NaN prefill), that
guard rows past the last row stay NaN, that the split-K tickets are back to zero and that a second launch is bitwise
identical.  Observed largest |err| / scale per variant go to $RB_PARITY_OBSERVED when that variable is set."""
import ctypes as C
import html
import json
import os
import re
import warnings

import numpy as np
import pytest
import torch

import head_ref as R
from test_gpu_parity import DEV, FakeEnv, make_args, synthetic_ring

pytestmark = pytest.mark.gpu

NAN = float("nan")
GUARD = 3                 # rows past the last one that must stay untouched


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


def stream():
    return torch.cuda.current_stream().cuda_stream


def record(key, value):
    """Largest observed |err| / scale per (variant, output), merged into $RB_PARITY_OBSERVED."""
    path = os.environ.get("RB_PARITY_OBSERVED")
    if not path:
        return
    data = json.load(open(path)) if os.path.exists(path) else {}
    data.setdefault("head_f64_tau", R.TAU)
    data.setdefault("head_f64_tau_tc", R.TAU_TC)
    data.setdefault("head_f64_tau_tc_wgrad", R.TAU_TC_WGRAD)
    data[key] = max(float(value), data.get(key, 0.0))
    with open(path, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)


def params_struct(p):
    from rainbow_b200 import _lib
    s = _lib.HeadParams()
    for k in R.PARAMS + R.FACTORS:
        for i in range(2):
            getattr(s, k)[i] = _lib.ptr(p[k][i]) if p[k] is not None else None
    s.conv_features, s.hidden, s.atoms, s.actions = p["K1"], p["H"], p["Z"], p["A"]
    return s


def grads_struct(g):
    from rainbow_b200 import _lib
    s = _lib.HeadGrads()
    for k in R.PARAMS:
        for i in range(2):
            getattr(s, k)[i] = _lib.ptr(g[f"{k}.{i}"])
    return s


def expected_variants(K1, H, m_lo, m_hi, debug):
    """Kernels rb_head_forward must launch.  Mirrors the host-side choice in rainbow_b200/csrc/rb_head.cu rb_head_forward
    (tensor-core layer 1 iff rbi::head_fc1_tc_ok in rb_head_tc.cu; single-pass layer 2 iff its shared memory
    (64 + 4) * (H + 4) floats fits in 200 KB) and the split of head_fc1_tc_splits (R.tc_splits); update them together."""
    tc = not (debug & 4) and (m_hi == 0 or m_lo % 8 == 0)
    split2 = bool(debug & 8) or (64 + 4) * (H + 4) * 4 > 200 * 1024
    return dict(fc1_tc=tc, fc1_ffma=not tc, reduce1=tc and R.tc_splits(K1, H)[0] > 1, fc2_single=not split2, fc2_splitk=split2)


_FC = re.compile(r"k_head_fc(?:<\s*\d+\s*,\s*(\d)\s*>|ILi\d+ELi(\d)E)")


def graph_kernels(fn, dot_path):
    """Run fn() under CUDA graph capture and return (graph, fn's result, text of the graph's DOT dump).  The dump lists
    the kernel of every node the launches recorded, so which variants rb_head_forward chose is read from the work itself
    -- not from profiler activity records, which can go missing.  The graph is replayed once before it is returned:
    fn's outputs then hold what the captured kernels computed."""
    g = torch.cuda.CUDAGraph(keep_graph=True)
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        out = fn()
    with warnings.catch_warnings():                                     # debug_dump announces itself with a warning
        warnings.simplefilter("ignore")
        g.debug_dump(str(dot_path))
    g.replay()
    torch.cuda.synchronize()
    return g, out, html.unescape(open(dot_path).read())


def variants_of(dot):
    layers = {int(a or b) for a, b in _FC.findall(dot)}
    return dict(fc1_tc="k_head_fc1_tc" in dot, fc1_ffma=1 in layers, reduce1="k_head_reduce1" in dot,
                fc2_single="k_head_fc2" in dot, fc2_splitk=2 in layers)


class Head:
    """Parameters of one head on the device plus the scratch its forward needs."""

    def __init__(self, K1, H, Z, A, noisy, seed):
        self.p = R.make_head(K1, H, Z, A, noisy, seed, DEV)
        self.K1, self.H, self.Z, self.A, self.ncols = K1, H, Z, A, Z * (1 + A)
        s1, s2 = C.c_int(), C.c_int()
        assert lib().rb_head_splits(K1, H, C.byref(s1), C.byref(s2)) == 0
        self.s1, self.s2 = s1.value, s2.value
        self.tickets = torch.zeros(lib().rb_head_ticket_count(), dtype=torch.int32, device=DEV)
        self.ps = params_struct(self.p)

    def forward(self, x_lo, x_hi, debug=0):
        M = x_lo.shape[0] + (0 if x_hi is None else x_hi.shape[0])
        part1 = torch.full((self.s1, M, 2 * self.H), NAN, device=DEV)
        part2 = torch.full((self.s2, M, self.ncols), NAN, device=DEV)
        h = torch.full((M + GUARD, 2 * self.H), NAN, device=DEV)
        z = torch.full((M + GUARD, self.ncols), NAN, device=DEV)
        L = lib()
        assert L.rb_head_debug(debug) == 0
        try:
            rc = L.rb_head_forward(C.byref(self.ps), x_lo.data_ptr(), x_lo.shape[0], None if x_hi is None else x_hi.data_ptr(),
                                   0 if x_hi is None else x_hi.shape[0], part1.data_ptr(), part2.data_ptr(), self.tickets.data_ptr(),
                                   h.data_ptr(), z.data_ptr(), stream())
        finally:
            L.rb_head_debug(0)
        assert rc == 0, L.rb_last_error()
        return h, z


def assert_guard_nan(name, t, rows):
    assert torch.isnan(t[rows:]).all(), f"{name}: written past its last row"


# ---------------------------------------------------------------------------------------------------------------------
# forward, logits, q_values
AZ = [(1, 51), (6, 51), (18, 51), (6, 101), (18, 101), (1, 101)]


def _fwd_cases():
    cases = []   # (K1, H, A, Z, noisy, m_lo, m_hi, debug)
    i = 0
    for K1 in (32, 64, 576, 3136):                                     # shape grid, both modes
        for H in (64, 128, 512, 1024, 2048):
            A, Z = AZ[i % len(AZ)]
            i += 1
            for noisy in (True, False):
                cases.append((K1, H, A, Z, noisy, 33, 0, 0))
    for K1, H, A, Z in ((3136, 512, 6, 51), (576, 1024, 18, 51)):    # row tiles up to FusedHead.MAX_ROWS
        for j, M in enumerate((1, 8, 31, 32, 33, 64, 65, 100, 257, 4096)):
            cases.append((K1, H, A, Z, j % 2 == 0, M, 0, 0))
        for B in (8, 16, 32, 2048):                                    # [s; s'] row blocks: tensor-core path
            cases.append((K1, H, A, Z, True, B, B, 0))
        for m_lo, m_hi in ((7, 7), (33, 32), (50, 50)):                # m_lo % 8 != 0: FFMA fallback
            cases.append((K1, H, A, Z, True, m_lo, m_hi, 0))
    for K1, H, A, Z in ((3136, 512, 6, 51), (576, 256, 18, 51), (3136, 2048, 6, 101), (32, 512, 6, 51)):   # the other variant
        for debug in (4, 8, 12):
            cases.append((K1, H, A, Z, True, 32, 32, debug))
    return cases


FWD_CASES = _fwd_cases()


def _fwd_id(c):
    K1, H, A, Z, noisy, m_lo, m_hi, debug = c
    return f"K{K1}-H{H}-A{A}-Z{Z}-{'noisy' if noisy else 'eval'}-m{m_lo}+{m_hi}" + (f"-dbg{debug}" if debug else "")


@pytest.mark.parametrize("case", FWD_CASES, ids=[_fwd_id(c) for c in FWD_CASES])
def test_head_forward_f64(case, tmp_path):
    K1, H, A, Z, noisy, m_lo, m_hi, debug = case
    M = m_lo + m_hi
    seed = hash(case) & 0xFFFF
    hd = Head(K1, H, Z, A, noisy, seed)
    x = R.make_features(M, K1, seed + 1, DEV)
    x_lo = x[:m_lo].clone()
    x_hi = x[m_lo:].clone() if m_hi else None
    h1, z1 = hd.forward(x_lo, x_hi, debug)                             # eager launch
    graph, (h, z), dot = graph_kernels(                                # graph: keeps h, z (its memory pool) alive
        lambda: hd.forward(x_lo, x_hi, debug), tmp_path / "forward.dot")
    assert "k_head_" in dot, "the graph dump names no head kernel: " + dot[:2000]
    want = expected_variants(K1, H, m_lo, m_hi, debug)
    ran = variants_of(dot)
    assert ran == want, f"kernels launched {ran}, expected {want}"
    assert int(hd.tickets.abs().sum()) == 0, "split-K tickets are left at zero"
    assert_guard_nan("h", h, M)
    assert_guard_nan("z", z, M)
    assert torch.equal(h1[:M], h[:M]) and torch.equal(z1[:M], z[:M]), "a second launch is bitwise identical"
    h, z = h[:M], z[:M]
    l1 = "fc1_tc" if want["fc1_tc"] else "fc1_ffma"
    l2 = "fc2_splitk" if want["fc2_splitk"] else "fc2_single"
    pre, s1 = R.layer1(hd.p, x)
    record(f"{l1}.h", R.assert_within(f"h ({l1})", h, pre.relu(), s1, R.TAU_TC if want["fc1_tc"] else R.TAU))
    z_ref, s2 = R.layer2(hd.p, h)
    record(f"{l2}.z", R.assert_within(f"z ({l2})", z, z_ref, s2))

    L = lib()
    q = torch.full((M + GUARD, A, Z), NAN, device=DEV)
    assert L.rb_head_logits(z.data_ptr(), M, A, Z, q.data_ptr(), stream()) == 0
    assert_guard_nan("logits", q, M)
    q_ref, sq = R.logits(z, A, Z)
    record("logits.q", R.assert_within("logits", q[:M], q_ref, sq))

    support = torch.linspace(-10, 10, Z, device=DEV)
    ev = torch.full((M + GUARD, A), NAN, device=DEV)
    best_a = torch.full((M + GUARD,), -7, dtype=torch.int64, device=DEV)
    best_q = torch.full((M + GUARD,), NAN, device=DEV)
    assert L.rb_q_values(z.data_ptr(), M, A, Z, support.data_ptr(), ev.data_ptr(), best_a.data_ptr(), best_q.data_ptr(),
                         stream()) == 0
    assert_guard_nan("q_values", ev, M)
    assert_guard_nan("best_q", best_q, M)
    assert bool((best_a[M:] == -7).all()), "best_action: written past its last row"
    ev_ref, sev = R.q_values(z, A, Z, support)
    record("q_values.ev", R.assert_within("q_values", ev[:M], ev_ref, sev))
    bound = R.TAU * sev.max(1).values
    top2 = ev_ref.topk(min(2, A), dim=1).values
    clear = (top2[:, 0] - top2[:, -1] > 2 * bound) if A > 1 else torch.ones(M, dtype=torch.bool, device=DEV)
    assert bool((best_a[:M][clear] == ev_ref.argmax(1)[clear]).all()), "arg-max where the top two values are apart"
    R.assert_within("best_q", best_q[:M], ev_ref.max(1).values, sev.max(1).values)


# ---------------------------------------------------------------------------------------------------------------------
# backward
BWD_AZ = [(3, 51), (6, 51), (18, 51), (18, 59), (6, 101)]


def _bwd_cases():
    cases = []   # (K1, H, A, Z, B, relu_mask_x, noisy)
    i = 0
    for B in (1, 7, 8, 17, 31, 32):
        for H in (64, 512, 1024):
            A, Z = BWD_AZ[i % len(BWD_AZ)]
            K1 = (576, 3136, 64)[i % 3]
            cases.append((K1, H, A, Z, B, i % 2 == 1, (i // 2) % 2 == 0))
            i += 1
    for A, Z in BWD_AZ:                                                 # every (A, Z) at hidden 1024, all four flag pairs
        for relu, noisy in ((True, True), (False, False), (True, False), (False, True)):
            cases.append((576, 1024, A, Z, 32, relu, noisy))
    return cases


BWD_CASES = _bwd_cases()


def _bwd_id(c):
    K1, H, A, Z, B, relu, noisy = c
    return f"K{K1}-H{H}-A{A}-Z{Z}-B{B}-{'relu' if relu else 'norelu'}-{'noisy' if noisy else 'eval'}"


@pytest.mark.parametrize("case", BWD_CASES, ids=[_bwd_id(c) for c in BWD_CASES])
def test_head_backward_f64(case):
    K1, H, A, Z, B, relu, noisy = case
    seed = hash(case) & 0xFFFF
    hd = Head(K1, H, Z, A, noisy, seed)
    x = R.make_features(B, K1, seed + 1, DEV)
    h, _ = hd.forward(x, None)
    h = h[:B].contiguous()
    g = torch.Generator(device=DEV).manual_seed(seed + 2)
    dz = torch.randn(B, hd.ncols, device=DEV, generator=g) * 0.1
    L = lib()

    def run():
        grads = {f"{k}.{s}": torch.full_like(hd.p[k][s], NAN) for k in R.PARAMS for s in range(2)}
        dh_s = torch.full(((B + 32) * 2 * H + GUARD,), NAN, device=DEV)     # dh [B][2H], dhT [2H][32], guard
        dx = torch.full((B + GUARD, K1), NAN, device=DEV)
        gs = grads_struct(grads)
        rc = L.rb_head_backward(C.byref(hd.ps), C.byref(gs), x.data_ptr(), h.data_ptr(), dz.data_ptr(), B, dh_s.data_ptr(),
                                dx.data_ptr(), 1 if relu else 0, 7, stream())
        assert rc == 0, L.rb_last_error()
        return grads, dh_s, dx

    grads, dh_s, dx = run()
    assert_guard_nan("dh scratch", dh_s, (B + 32) * 2 * H)
    assert_guard_nan("dx", dx, B)
    dh = dh_s[:B * 2 * H].view(B, 2 * H)
    dhT = dh_s[B * 2 * H:(B + 32) * 2 * H].view(2 * H, 32)
    assert torch.equal(dhT[:, :B], dh.T) and bool((dhT[:, B:] == 0).all()), "dhT is dh transposed, rows past B zero"
    ref2 = R.backward_layer2(hd.p, h, dz)
    ref1 = R.backward_layer1(hd.p, x, dh, relu)
    got = dict(grads, dh=dh, dx=dx[:B])
    for name, (ref, scale) in list(ref2.items()) + list(ref1.items()):
        tau = R.TAU_TC if name == "dx" else R.TAU_TC_WGRAD if name.startswith("w1_") else R.TAU   # k_head_bwd1's tensor-core products
        record(f"bwd.{name.split('.')[0]}", R.assert_within(name, got[name], ref, scale, tau))

    grads2, dh_s2, dx2 = run()
    n = (B + 32) * 2 * H                                                # the NaN guard compares unequal to itself
    assert torch.equal(dx2[:B], dx[:B]) and torch.equal(dh_s2[:n], dh_s[:n])
    for k in grads:
        assert torch.equal(grads2[k], grads[k]), f"{k}: a second launch is bitwise identical"


def test_backward_cases_reach_the_dh_eps_out_fallback():
    """k_head_dh keeps 8 eps_out factors per thread in registers (DH_MAXI); actions * atoms > 1024 needs the load past them."""
    assert any(A * Z * 2 > 8 * 256 and noisy for _, _, A, Z, _, _, noisy in BWD_CASES)
    assert any(H == 1024 for _, H, *_ in BWD_CASES)


# ---------------------------------------------------------------------------------------------------------------------
# one predicate for the shapes the fused head takes
@pytest.mark.parametrize("H", [64, 1024, 1088, 2048])
def test_head_supported_agrees_with_the_calls(H):
    """rb_head_supported(conv_features, hidden, atoms, actions, rows, backward_batch) returns what rb_head_forward over
    `rows` rows and rb_head_backward over `backward_batch` rows return (with valid pointers)."""
    L = lib()
    K1 = 32
    for A, Z in ((18, 59), (18, 60), (10, 101), (11, 101), (18, 101), (6, 51)):
        hd = Head(K1, H, Z, A, True, 5)
        for rows in (64, 4096):
            want = L.rb_head_supported(K1, H, Z, A, rows, 0)
            x = R.make_features(rows, K1, 6, DEV)
            part1 = torch.empty(hd.s1 * rows * 2 * H, device=DEV)
            part2 = torch.empty(hd.s2 * rows * hd.ncols, device=DEV)
            h = torch.empty(rows, 2 * H, device=DEV)
            z = torch.empty(rows, hd.ncols, device=DEV)
            got = L.rb_head_forward(C.byref(hd.ps), x.data_ptr(), rows, None, 0, part1.data_ptr(), part2.data_ptr(),
                                    hd.tickets.data_ptr(), h.data_ptr(), z.data_ptr(), stream())
            assert got == want, (A, Z, rows, got, want)
        B = 32
        want = L.rb_head_supported(K1, H, Z, A, 0, B)
        x = R.make_features(B, K1, 7, DEV)
        h = torch.rand(B, 2 * H, device=DEV)
        dz = torch.randn(B, hd.ncols, device=DEV)
        grads = {f"{k}.{s}": torch.full_like(hd.p[k][s], NAN) for k in R.PARAMS for s in range(2)}
        dh_s = torch.empty((B + 32) * 2 * H, device=DEV)
        dx = torch.empty(B, K1, device=DEV)
        for parts in (1, 2, 4, 7):
            got = L.rb_head_backward(C.byref(hd.ps), C.byref(grads_struct(grads)), x.data_ptr(), h.data_ptr(), dz.data_ptr(), B,
                                     dh_s.data_ptr(), dx.data_ptr(), 1, parts, stream())
            assert got == want, (A, Z, parts, got, want)
        if want != 0:
            assert all(bool(torch.isnan(t).all()) for t in grads.values()), "a refused backward writes nothing"
    torch.cuda.synchronize()


def _batch(B, A, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.arange(B, device=DEV), torch.rand(B, 4, 84, 84, device=DEV, generator=g),
            torch.randint(0, A, (B,), device=DEV, generator=g), torch.rand(B, device=DEV, generator=g) * 4 - 2,
            torch.rand(B, 4, 84, 84, device=DEV, generator=g), (torch.rand(B, 1, device=DEV, generator=g) > 0.2).float(),
            torch.rand(B, device=DEV, generator=g) * 0.8 + 0.2)


@pytest.mark.parametrize("hidden,A,Z,fused", [(64, 18, 101, False), (2048, 6, 51, False), (64, 18, 59, True)],
                         ids=["A18-Z101", "hidden2048", "A18-Z59"])
def test_learner_takes_the_library_path_where_the_fused_backward_refuses(hidden, A, Z, fused):
    """Agent._fused_path asks rb_head_supported for the backward too: shapes whose fused backward returns RB_ERR_RANGE
    (actions * atoms too large for the dh kernel, hidden > 1024) update on the library path -- same result as
    use_fused_head=False -- instead of raising on the first update; (A 18, Z 59) still takes the fused path.  Acting keeps
    the fused forward at all three shapes."""
    from rainbow_b200 import RainbowB200Error
    from rainbow_b200.agent import Agent
    B = 8

    def agent(**kw):
        torch.manual_seed(0)
        args = make_args(batch_size=B, architecture="data-efficient", hidden_size=hidden, atoms=Z, cuda_graph=False, **kw)
        return Agent(args, FakeEnv(A))

    ag = agent()
    assert ag._fused_path(B) == fused
    assert ag.online_net.fused_ok(64)
    batch = _batch(B, A, 1)
    if not fused:
        forced = agent()
        forced._fused_path = lambda b: True        # what the learner chose before it asked about the backward
        with pytest.raises(RainbowB200Error, match="error -34"):
            forced._update_from_batch(batch)
        torch.cuda.synchronize()
        ref = agent(fused_head=False)
        loss_ref = ref._update_from_batch(batch)
    loss = ag._update_from_batch(batch)
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all()
    if not fused:
        torch.testing.assert_close(loss, loss_ref, rtol=1e-6, atol=0)
        torch.testing.assert_close(ag.optimiser.flat_param, ref.optimiser.flat_param, rtol=0, atol=1e-8)
    mem, _ = synthetic_ring(4096)
    ag.learn(mem)
    torch.cuda.synchronize()
    assert torch.isfinite(ag.last_loss).all()
    with torch.no_grad():
        a, v = ag.q_select(torch.rand(3, 4, 84, 84, device=DEV))
    assert bool(((a >= 0) & (a < A)).all()) and torch.isfinite(v).all()
