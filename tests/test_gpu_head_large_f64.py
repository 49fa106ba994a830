"""The large-batch backward of the fused noisy dueling head (rb_head_backward with the layer-1 kernels it runs above 32
rows: k_head_wgrad2, k_head_dh over 32-row batch tiles, k_head_bwd1_wgrad, k_head_bwd1_dx; rb_head_debug bit 4 makes it
run them at every B) through its C ABI against the float64 reference of tests/head_ref.py, per element
(|err| <= tau * scale), in the harness style of tests/test_gpu_head_f64.py:

 * B in {1, 31, 32, 33, 64, 100, 255, 256, 511, 512} x hidden {64, 512, 1024}, conv_features cycling {576, 3136, 64},
   (actions, atoms) cycling BWD_AZ (actions * atoms up to 1062: the dh kernel's eps_out fallback), all ReLU-mask / eval
   combinations, and C4's learner shape (3136 / 512 / 6 / 51 / B 512);
 * NaN-prefilled outputs, guard rows past B, the dhT layout [2H][round_up(B, 32)] with its zero columns, a second launch
   and a CUDA-graph replay bitwise identical to an eager launch, the kernels read from the graph's kernel nodes;
 * without the debug bit the call runs these kernels above 32 rows, with the same outputs bitwise, and k_head_bwd1 at
   B <= 32: dh and dhT bitwise equal, the other outputs within tau;
 * rb_head_supported agrees with the call up to and past B 512, and a refused call writes nothing;
 * the learner at batch 512 against the unmodified reference (tests/golden/update_c4.npz, oracle/gen_update_c4.py),
   graph replay == eager at batch 64 and 512, and the shapes whose fused backward is refused updating on the library path.
The tensor-core bounds are TAU_LARGE_WGRAD / TAU_LARGE_DX of tests/test_large_batch_tf32_numerics.py.  Observed largest
|err| / scale go to $RB_PARITY_OBSERVED when that variable is set."""
import ctypes as C
import hashlib
import re

import numpy as np
import pytest
import torch

import head_ref as R
from test_gpu_head_f64 import BWD_AZ, GUARD, NAN, Head, _batch, assert_guard_nan, graph_kernels, grads_struct, lib, record, stream
from test_gpu_parity import DEV, FakeEnv, make_args, synthetic_ring
from test_large_batch_tf32_numerics import TAU_LARGE_DX, TAU_LARGE_WGRAD

pytestmark = pytest.mark.gpu

_SMALL_BWD1 = re.compile(r"k_head_bwd1(?:\(|E|\b(?!_))")   # k_head_bwd1 itself, not k_head_bwd1_wgrad / _dx


def bp(B):
    return -(-B // 32) * 32


def tau_of(name):
    return TAU_LARGE_DX if name == "dx" else TAU_LARGE_WGRAD if name.startswith("w1_") else R.TAU


def large_kernels_of(dot):
    return dict(wgrad2="k_head_wgrad2" in dot, dh="k_head_dh" in dot, wgrad1="k_head_bwd1_wgrad" in dot,
                dx="k_head_bwd1_dx" in dot, small_bwd1=bool(_SMALL_BWD1.search(dot)))


def backward(hd, x, h, dz, B, relu, large=True, parts=7):
    """One rb_head_backward launch into NaN-filled outputs; returns (rc, grads, dh scratch, dx).  large=True sets
    rb_head_debug bit 4 for the call (the large-batch layer-1 kernels at every B); large=False lets the call choose."""
    H, K1 = hd.H, hd.K1
    grads = {f"{k}.{s}": torch.full_like(hd.p[k][s], NAN) for k in R.PARAMS for s in range(2)}
    dh_s = torch.full(((B + bp(B)) * 2 * H + GUARD,), NAN, device=DEV)   # dh [B][2H], dhT [2H][Bp], guard
    dx = torch.full((B + GUARD, K1), NAN, device=DEV)
    L = lib()
    if large:
        L.rb_head_debug(16)
    try:
        rc = L.rb_head_backward(C.byref(hd.ps), C.byref(grads_struct(grads)), x.data_ptr(), h.data_ptr(), dz.data_ptr(), B,
                                dh_s.data_ptr(), dx.data_ptr(), 1 if relu else 0, parts, stream())
    finally:
        L.rb_head_debug(0)
    return rc, grads, dh_s, dx


def inputs(hd, B, seed):
    x = R.make_features(B, hd.K1, seed + 1, DEV)
    h, _ = hd.forward(x, None)
    h = h[:B].contiguous()
    g = torch.Generator(device=DEV).manual_seed(seed + 2)
    dz = torch.randn(B, hd.ncols, device=DEV, generator=g) * 0.1
    return x, h, dz


def _cases():
    cases = []   # (K1, H, A, Z, B, relu_mask_x, noisy)
    i = 0
    for B in (1, 31, 32, 33, 64, 100, 255, 256, 511, 512):
        for H in (64, 512, 1024):
            A, Z = BWD_AZ[i % len(BWD_AZ)]
            K1 = (576, 3136, 64)[i % 3]
            cases.append((K1, H, A, Z, B, i % 2 == 1, (i // 2) % 2 == 0))
            i += 1
    for relu, noisy in ((True, True), (False, False)):                   # C4's learner shape
        cases.append((3136, 512, 6, 51, 512, relu, noisy))
    return cases


CASES = _cases()


def _id(c):
    K1, H, A, Z, B, relu, noisy = c
    return f"K{K1}-H{H}-A{A}-Z{Z}-B{B}-{'relu' if relu else 'norelu'}-{'noisy' if noisy else 'eval'}"


def test_cases_cover_the_flags_and_the_dh_fallback():
    assert {(relu, noisy) for *_, relu, noisy in CASES} == {(a, b) for a in (True, False) for b in (True, False)}
    assert any(A * Z * 2 > 8 * 256 and noisy and B > 32 for _, _, A, Z, B, _, noisy in CASES)
    assert (3136, 512, 6, 51, 512, True, True) in CASES


@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_head_backward_large_f64(case, tmp_path):
    K1, H, A, Z, B, relu, noisy = case
    seed = hash(case) & 0xFFFF
    hd = Head(K1, H, Z, A, noisy, seed)
    x, h, dz = inputs(hd, B, seed)
    Bp, n = bp(B), (B + bp(B)) * 2 * H

    rc, grads, dh_s, dx = backward(hd, x, h, dz, B, relu)
    assert rc == 0, lib().rb_last_error()
    assert_guard_nan("dh scratch", dh_s, n)
    assert_guard_nan("dx", dx, B)
    dh = dh_s[:B * 2 * H].view(B, 2 * H)
    dhT = dh_s[B * 2 * H:n].view(2 * H, Bp)
    assert torch.equal(dhT[:, :B], dh.T) and bool((dhT[:, B:] == 0).all()), "dhT is dh transposed, columns past B zero"
    ref2 = R.backward_layer2(hd.p, h, dz)
    ref1 = R.backward_layer1(hd.p, x, dh, relu)
    got = dict(grads, dh=dh, dx=dx[:B])
    for name, (ref, scale) in list(ref2.items()) + list(ref1.items()):
        record(f"bwd_large.{name.split('.')[0]}", R.assert_within(name, got[name], ref, scale, tau_of(name)))

    _, grads2, dh_s2, dx2 = backward(hd, x, h, dz, B, relu)              # a second launch
    assert torch.equal(dx2[:B], dx[:B]) and torch.equal(dh_s2[:n], dh_s[:n])
    for k in grads:
        assert torch.equal(grads2[k], grads[k]), f"{k}: a second launch is bitwise identical"

    graph, (rc_g, grads_g, dh_g, dx_g), dot = graph_kernels(lambda: backward(hd, x, h, dz, B, relu), tmp_path / "bwd.dot")
    assert rc_g == 0
    ran = large_kernels_of(dot)
    assert ran == dict(wgrad2=True, dh=True, wgrad1=True, dx=True, small_bwd1=False), ran
    assert torch.equal(dx_g[:B], dx[:B]) and torch.equal(dh_g[:n], dh_s[:n]), "graph replay == eager launch"
    for k in grads:
        assert torch.equal(grads_g[k], grads[k]), f"{k}: graph replay == eager launch"

    # without the debug bit: the large-batch kernels above 32 rows, k_head_bwd1 at B <= 32 (same layer-2 kernels)
    _, (rc_d, grads_d, dh_d, dx_d), dot = graph_kernels(lambda: backward(hd, x, h, dz, B, relu, large=False),
                                                        tmp_path / "bwd_default.dot")
    assert rc_d == 0
    ran = large_kernels_of(dot)
    assert torch.equal(dh_d[:n], dh_s[:n]), "dh and dhT bitwise equal to the large-batch kernels' run"
    if B > 32:
        assert ran == dict(wgrad2=True, dh=True, wgrad1=True, dx=True, small_bwd1=False), ran
        assert torch.equal(dx_d[:B], dx[:B]), "the default call runs the same kernels"
        for k in grads:
            assert torch.equal(grads_d[k], grads[k]), f"{k}: the default call runs the same kernels"
    else:
        assert ran == dict(wgrad2=True, dh=True, wgrad1=False, dx=False, small_bwd1=True), ran
        refs = dict(list(ref2.items()) + list(ref1.items()))
        for k in grads:
            R.assert_within(f"{k} vs k_head_bwd1", grads[k], R._d(grads_d[k]), refs[k][1], tau_of(k))
        R.assert_within("dx vs k_head_bwd1", dx[:B], R._d(dx_d[:B]), refs["dx"][1], tau_of("dx"))


@pytest.mark.parametrize("H", [64, 1024, 1088, 2048])
def test_head_large_supported_agrees_with_the_call(H):
    """rb_head_supported(conv_features, hidden, atoms, actions, 0, B) returns what rb_head_backward returns with valid
    pointers at batch sizes past k_head_bwd1's 32 rows, for every `parts`; a refused call leaves its NaN-filled outputs
    untouched."""
    L = lib()
    K1 = 32
    for A, Z in ((18, 59), (18, 60), (11, 101), (6, 51)):
        hd = Head(K1, H, Z, A, True, 5)
        for B in (33, 512, 513):
            want = L.rb_head_supported(K1, H, Z, A, 0, B)
            x = R.make_features(B, K1, 7, DEV)
            h = torch.rand(B, 2 * H, device=DEV)
            dz = torch.randn(B, hd.ncols, device=DEV)
            for parts in (1, 2, 4, 7):
                got, grads, dh_s, dx = backward(hd, x, h, dz, B, True, large=False, parts=parts)
                assert got == want, (A, Z, B, parts, got, want)
                if want != 0:
                    torch.cuda.synchronize()
                    assert all(bool(torch.isnan(t).all()) for t in grads.values()), "a refused call writes nothing"
                    assert bool(torch.isnan(dh_s).all()) and bool(torch.isnan(dx).all()), "a refused call writes nothing"
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# the learner at batch sizes above 32
def _tree_from_leaves(leaves, tree_start):
    """The reference's sum tree from its leaves (every node the float32 sum of its children; oracle/gen_update_c4.py)."""
    tree = np.zeros(tree_start + leaves.size, np.float32)
    tree[tree_start:] = leaves
    lo = tree_start
    while lo > 0:
        plo = (lo - 1) // 2
        par = np.arange(plo, lo)
        tree[par] = tree[2 * par + 1] + tree[2 * par + 2]
        lo = plo
    return tree


def test_update_c4_vs_reference():
    """Three `reset_noise(); learn(mem)` pairs at batch 512 (canonical / 512, n 3, 6 actions, 16384 transitions) against
    the unmodified reference's trajectory (tests/golden/update_c4.npz, written by oracle/gen_update_c4.py), with the bounds
    of test_gpu_update.py::test_full_update_vs_reference: sampled indices bit-exact, loss 1e-5, gradients 1e-6 (conv 2e-6),
    parameters 1e-7 (conv 2e-7), priority leaves == fl32(sqrt(loss)), the tree after the reference's write-back bit-exact
    (SHA-256 of the whole tree).  The update must take the fused path with the large-batch layer-1 kernels.

    cuDNN runs its deterministic algorithms here.  With its default conv backward the conv weights after step 0 differ in
    their last bits from run to run; at batch 512 a step then walks 1.5 M head-ReLU pre-activations, and one of them can land
    on the other side of zero than in the reference, moving that unit's bias gradient by |dh| (observed on an H100: one run
    in three, fc_h_a bias 1.3e-6 at step 1; the other runs 2.2e-7, the same as every deterministic run)."""
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    try:
        _update_c4_vs_reference()
    finally:
        torch.backends.cudnn.deterministic = old


def _update_c4_vs_reference():
    import json
    import os

    from helpers import assert_bits_equal, golden, update_case_ring
    from rainbow_b200 import _lib
    from rainbow_b200.agent import Agent
    from rainbow_b200.memory import ReplayMemory
    g = golden("update_c4")
    case = {k[5:]: g[k].item() if g[k].ndim == 0 else g[k].tolist() for k in g if k.startswith("case_")}
    torch.manual_seed(case["seed"])                     # same host RNG stream as the reference's Agent construction
    args = make_args(batch_size=case["B"], multi_step=case["n"], architecture=case["arch"], hidden_size=case["hidden"],
                     cuda_graph=False)
    ag = Agent(args, FakeEnv(case["A"]))
    on, tg = ag.online_net, ag.target_net
    sd0 = torch.cat([p.detach().reshape(-1).cpu() for _, p in on.named_parameters()]).numpy()
    assert hashlib.sha256(sd0.tobytes()).hexdigest() == case["sd0_sha"], "initial parameters differ from the reference's"
    assert ag._fused_path(case["B"])
    mem = ReplayMemory(args, case["cap"], rng="numpy")
    meta, ts = g["ring_meta"], case["tree_start"]
    mem.transitions.load_arrays(_tree_from_leaves(g["ring_leaves"], ts), update_case_ring(case).reshape(case["cap"], -1),
                                g["ring_timestep"], g["ring_action"], g["ring_reward"], g["ring_nonterminal"], int(meta[0]),
                                bool(meta[1]), int(meta[2]), float(g["ring_max"]))
    mem.t = int(meta[2])
    tr = mem.transitions
    # the reference's noise draws: torch.randn on the CPU generator from its state after the Agent was built
    gen = torch.Generator()
    gen.set_state(torch.from_numpy(g["rng_state"]))
    draws = [torch.randn(int(n), generator=gen) for n in g["draw_sizes"]]
    strides = dict(zip(g["param_names"].tolist(), g["param_strides"].tolist()))
    np.random.seed(case["seed"] + 100)                  # the stream the reference's mem.sample consumed (memory.py:129)
    obs = dict(loss=0.0, grad=0.0, param=0.0, param_head=0.0)
    bad = []

    def dev(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)

    def noise(i):                                       # 8 draws per net and step: eps_in, eps_out per layer in reset order
        d = draws[8 * i:8 * i + 8]
        return dev(torch.cat(d[0::2]).numpy()), dev(torch.cat(d[1::2]).numpy())

    def close(a, b, atol, what):
        d = float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())
        if not d <= atol:
            bad.append(f"{what}: max |diff| {d:.3e} > {atol:.1e}")
        return d

    with _lib.KernelTimer() as kt:
        for k in range(case["steps"]):
            on.queue_noise(*noise(2 * k))
            ag.reset_noise()                                                   # main.py:150
            tg.queue_noise(*noise(2 * k + 1))
            tree_before, max_before = tr.tree.clone(), tr.running_max.clone()
            ag.learn(mem)                                                      # main.py:151
            torch.cuda.synchronize()
            assert not tg._noise_queue and not on._noise_queue
            tidx = mem._last.tree_idx.cpu().numpy()
            assert np.array_equal(tidx, g[f"s{k}_tidx"]), f"step {k}: sampled indices differ"
            loss = ag.last_loss.cpu().numpy()
            obs["loss"] = max(obs["loss"], close(loss, g[f"s{k}_loss"], 1e-5, f"step {k} loss"))
            tree = tr.tree.cpu().numpy()
            assert len(set(tidx.tolist())) == len(tidx)
            assert_bits_equal(tree[tidx], np.sqrt(loss.astype(np.float32)), f"step {k}: leaf != sqrt(loss)")
            for key, p in on.named_parameters():
                st, conv = strides[key], key.startswith("convs")
                gr = p.grad.detach().cpu().numpy().reshape(-1)
                obs["grad"] = max(obs["grad"], close(gr[::st], g[f"s{k}_grad.{key}"], 2e-6 if conv else 1e-6, f"step {k} grad {key}"))
                s1, s2 = g[f"s{k}_gradsum.{key}"]
                assert abs(float(gr.astype(np.float64).sum()) - s1) <= 1e-5 * gr.size ** 0.5 + 2e-3 * abs(s1), f"step {k} grad sum {key}"
                assert abs(float((gr.astype(np.float64) ** 2).sum()) - s2) <= 2e-4 * s2 + 1e-12, f"step {k} grad sq sum {key}"
                pv = p.detach().cpu().numpy().reshape(-1)
                d = close(pv[::st], g[f"s{k}_param.{key}"], 2e-7 if conv else 1e-7, f"step {k} param {key}")
                obs["param"] = max(obs["param"], d)
                if not conv:
                    obs["param_head"] = max(obs["param_head"], d)
                assert abs(float(pv.astype(np.float64).sum()) - g[f"s{k}_paramsum.{key}"][0]) <= 2e-7 * pv.size
            assert int(ag.optimiser.step_count.item()) == k + 1
            # tree after the REFERENCE's write-back (same leaves, the reference's losses): bit-exact, incl. the running max
            tr.tree.copy_(tree_before)
            tr.running_max.copy_(max_before)
            mem.update_priorities(g[f"s{k}_tidx"], g[f"s{k}_loss"])
            torch.cuda.synchronize()
            tree = tr.tree.cpu().numpy()
            assert_bits_equal(tree[g[f"s{k}_tidx"]], g[f"s{k}_tree_leaves"], f"step {k}: written leaves")
            assert hashlib.sha256(np.ascontiguousarray(tree).tobytes()).hexdigest() == str(g[f"s{k}_tree_sha"]), \
                f"step {k}: tree after write-back differs from the reference's"
            assert np.float32(tr.max) == g[f"s{k}_max_after"]
    path = os.environ.get("RB_PARITY_OBSERVED")
    if path:
        data = json.load(open(path)) if os.path.exists(path) else {}
        data["full_update_c4"] = obs
        with open(path, "w") as f:
            json.dump(data, f, indent=1, sort_keys=True)
    assert not bad, "\n".join(bad)
    ran = set(kt.result)
    assert {"head_bwd1_wgrad", "head_bwd1_dx", "head_dh", "c51_dueling"} <= ran, ran
    assert "head_bwd1" not in ran and "c51" not in ran, ran


def _agent(B, **kw):
    from rainbow_b200.agent import Agent
    torch.manual_seed(5)
    return Agent(make_args(batch_size=B, **kw), FakeEnv(6))


@pytest.mark.parametrize("B", [64, 512])
def test_large_batch_update_graph_has_the_new_kernels(B, tmp_path):
    """One fused update at batch B captured as a CUDA graph: its kernel nodes include the large-batch layer-1 kernels and
    not k_head_bwd1."""
    ag = _agent(B, cuda_graph=False)
    assert ag._fused_path(B)
    batch = _batch(B, 6, 3)
    ag._update_from_batch(batch)                  # warm-up (cuDNN plans, scratch) outside the capture
    torch.cuda.synchronize()
    _, loss, dot = graph_kernels(lambda: ag._update_from_batch(batch), tmp_path / "update.dot")
    ran = large_kernels_of(dot)
    assert ran["wgrad1"] and ran["dx"] and ran["dh"] and not ran["small_bwd1"], ran
    assert torch.isfinite(loss).all()


@pytest.mark.parametrize("B", [64, 512])
def test_large_batch_graph_replay_equals_eager_bitwise(B):
    """2 eager warm-up updates + capture + replays leave parameters, Adam moments, priorities and losses bit-identical to
    the same number of eager updates, at batch sizes that run the large-batch layer-1 kernels (cuDNN deterministic)."""
    def trajectory(use_graph, steps=6):
        ag = _agent(B, cuda_graph=use_graph)
        mem, _ = synthetic_ring(16384, seed=3, args=dict(batch_size=B))
        mem.seed = 99
        losses = []
        for _ in range(steps):
            ag.reset_noise()
            ag.learn(mem)
            losses.append(ag.last_loss.clone())
        torch.cuda.synchronize()
        assert (ag._graph is not None) == use_graph
        assert ag._fused_path(B)
        return ag.optimiser.flat_param.clone(), mem.transitions.tree.clone(), torch.stack(losses), ag.optimiser.exp_avg_sq.clone()

    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    try:
        pe, te, le, ve = trajectory(False)
        pg, tg, lg, vg = trajectory(True)
    finally:
        torch.backends.cudnn.deterministic = old
    assert torch.equal(le, lg), "per-sample losses differ between graph replay and eager"
    assert torch.equal(te, tg), "sum trees differ"
    assert torch.equal(ve, vg) and torch.equal(pe, pg), "parameters / moments differ"


@pytest.mark.parametrize("B,hidden,A,Z", [(513, 512, 6, 51), (64, 2048, 6, 51), (64, 64, 18, 101)],
                         ids=["B513", "hidden2048", "A18-Z101"])
def test_large_batch_library_path_where_the_fused_backward_refuses(B, hidden, A, Z):
    """Batch 513, hidden 2048 and (A 18, Z 101) are outside rb_head_backward: the learner updates them on the library
    path, with the same result as fused_head=False, without raising."""
    from rainbow_b200.agent import Agent

    def agent(**kw):
        torch.manual_seed(0)
        args = make_args(batch_size=B, architecture="data-efficient", hidden_size=hidden, atoms=Z, cuda_graph=False, **kw)
        return Agent(args, FakeEnv(A))

    ag = agent()
    assert not ag._fused_path(B)
    batch = _batch(B, A, 1)
    loss = ag._update_from_batch(batch)
    ref = agent(fused_head=False)
    loss_ref = ref._update_from_batch(batch)
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all()
    torch.testing.assert_close(loss, loss_ref, rtol=1e-6, atol=0)
    torch.testing.assert_close(ag.optimiser.flat_param, ref.optimiser.flat_param, rtol=0, atol=1e-8)
