"""Bootstrapping through time-limit truncations, host side: the switch and its refusals, the new C entries' argument
checks (no launch is reached, so no GPU is needed), and tests/trunc_ref.py's statement of the truncation-aware gather
against the oracle's fixed-horizon gather at n = k, over history 1 and 4, n = 1, 3, 20 and 36 (a window past 32 records),
every cut k in 1 .. n - 1, a final observation at the ring's wrap and two short episodes in one window."""
import ctypes as C
import re

import numpy as np
import pytest
import torch

import oracle
import trunc_ref
from helpers import assert_bits_equal

RB_ERR_INVAL, RB_ERR_RANGE = -22, -34
SIZE = 2048
GAMMA = 0.97


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


# ---- the switch and its refusals ------------------------------------------------------------------------------------------
def bare_memory(switch, nonterminal=None):
    """A ReplayMemory without device state: enough for the checks that run before anything touches the ring."""
    from rainbow_b200.memory import ReplayMemory

    class Ring:
        pass

    mem = ReplayMemory.__new__(ReplayMemory)
    mem.bootstrap_truncation, mem._queue, mem.defer_appends = switch, [], False
    mem.transitions = Ring()
    mem.transitions.nonterminal = torch.as_tensor(np.zeros(8, np.uint8) if nonterminal is None else nonterminal)
    return mem


def test_append_truncated_needs_the_switch():
    from rainbow_b200._lib import RainbowB200Error
    mem = bare_memory(False)
    state = torch.zeros(4, 84, 84)
    with pytest.raises(RainbowB200Error, match="bootstrap_truncation"):
        mem.append_truncated(state, 1, 1.0, state)


def test_reference_pickle_refuses_final_records(tmp_path):
    from rainbow_b200._lib import RainbowB200Error
    from rainbow_b200.memory import save_reference_pickle
    mem = bare_memory(True, np.array([1, 1, 0, 1, 2, 0, 1, 1], np.uint8))
    assert mem.holds_final_records()
    with open(tmp_path / "mem.pkl", "wb") as f, pytest.raises(RainbowB200Error, match="final-observation records"):
        save_reference_pickle(mem, f)
    assert not bare_memory(True, np.array([1, 1, 0, 1, 1, 0, 1, 1], np.uint8)).holds_final_records()


def test_fixed_row_gamma_k_is_the_gamma_n_of_k_steps():
    """The kernels read gamma_k from the row's gamma_pow[k]; that must be the gamma_n the learner would use for a horizon of
    k steps, fl32(gamma ** k) -- for the replay's constant row and for every row of an annealed schedule."""
    from rainbow_b200.horizon import horizon_table
    for g in (0.99, 0.97, 0.9, 0.5, 0.997, 1.0, 0.0):
        for n in (1, 3, 20, 36, 63):
            row = horizon_table(1, n, n, g, g)[0]
            assert row["n"] == n and row["gamma_n"] == np.float32(g ** n)
            for k in range(1, n):
                assert row["gamma_pow"][k] == np.float32(g ** k) == np.float32(float(np.float32(g ** k)))
    rows = horizon_table(50, 10, 3, 0.97, 0.997)
    for r in rows:
        g_n = r["gamma_n"]
        for k in range(1, r["n"]):
            assert r["gamma_pow"][k] > g_n or r["gamma_pow"][k] == g_n == 0


def test_checkpoint_refuses_final_records_into_a_replay_without_the_switch():
    """load() refuses a manifest whose replay holds final-observation records before any other replay check or write."""
    from rainbow_b200 import checkpoint
    from rainbow_b200._lib import RainbowB200Error

    class Sync:
        world_size, rank, enabled = 1, 0, False

    class Agent:
        sync = Sync()

    man = dict(world_size=1, rank=0, save_id=5, structure=dict(replay={}), replay=dict(final_records=True))
    mem = bare_memory(False)
    import unittest.mock as um
    with um.patch.object(checkpoint, "_structure", lambda agent, mem: {}), \
            pytest.raises(RainbowB200Error, match="final-observation records"):
        agent = Agent()
        agent.distribution, agent.value_transform, agent.value_transform_eps = "categorical", None, None
        agent.quantile_average_copies, agent.munchausen, agent.risk = False, None, None
        checkpoint._validate(agent, mem, man)


# ---- the C entries: declarations, bindings and host-side refusals ---------------------------------------------------------
def header_decl(name):
    from rainbow_b200._build import HDR
    src = open(HDR).read()
    m = re.search(r"\bint " + name + r"\(([^;]*)\);", src)
    assert m, name
    return [a.strip() for a in m.group(1).replace("\n", " ").split(",")]


@pytest.mark.parametrize("new,old", [("rb_gather_trunc", "rb_gather_horizon"),
                                     ("rb_append_batch_trunc", "rb_append_batch")])
def test_entries_are_declared_and_bound_like_their_siblings(new, old):
    from rainbow_b200._lib import SIGNATURES
    assert header_decl(new) == header_decl(old)
    assert SIGNATURES[new] == SIGNATURES[old]
    assert len(SIGNATURES[new][1]) == len(header_decl(new))
    from rainbow_b200._build import HDR
    assert "#define RB_NONTERMINAL_FINAL 2" in open(HDR).read()


def gather_trunc_call(H=4, n=3, B=4, current=1, pad=0, intensity=0.0, m=1, k=1, frames=1, ctr=None, shifts=None):
    return lib().rb_gather_trunc(frames, 1, 1, 1, 1, 64, 1, B, H, n, current, 1, 1, 1, 1, 1, pad, intensity, m, k, 0, ctr,
                                 shifts, None, None)


def test_gather_trunc_refusals():
    L = lib()
    for kw, code in ((dict(current=None), RB_ERR_INVAL), (dict(frames=None), RB_ERR_INVAL),
                     (dict(H=32, n=33), RB_ERR_RANGE), (dict(B=65536), RB_ERR_RANGE), (dict(n=0), RB_ERR_INVAL),
                     (dict(pad=17), RB_ERR_RANGE), (dict(intensity=0.6), RB_ERR_RANGE),
                     (dict(intensity=float("nan")), RB_ERR_RANGE), (dict(m=9), RB_ERR_RANGE),
                     (dict(pad=4), RB_ERR_INVAL), (dict(pad=4, ctr=1), RB_ERR_INVAL)):
        assert gather_trunc_call(**kw) == code, kw
        assert L.rb_last_error().decode().startswith("rb_gather_trunc:"), (kw, L.rb_last_error())


def test_append_batch_trunc_refusals():
    L = lib()
    frames = (C.c_void_p * 1)(16)
    acts, rews, terms = (C.c_int32 * 1)(0), (C.c_float * 1)(0.0), (C.c_int32 * 1)(2)
    base = [1, 1023, 1024, 1, 1, 1, 1, 1, 1, 1, frames, acts, rews, terms, 1, None]
    for i, v, code in ((0, None, RB_ERR_INVAL), (2, 1023, RB_ERR_INVAL), (14, 0, RB_ERR_RANGE), (14, 9, RB_ERR_RANGE),
                       (10, (C.c_void_p * 1)(8), RB_ERR_INVAL)):
        args = list(base)
        args[i] = v
        assert L.rb_append_batch_trunc(*args) == code, (i, v)
        assert L.rb_last_error().decode().startswith("rb_append_batch_trunc:"), L.rb_last_error()


# ---- trunc_ref against the oracle's fixed-horizon gather ------------------------------------------------------------------
def base_ring(seed):
    """Random frames, actions and rewards; episodes of 5 to 60 records, each ending in a terminal."""
    rs = np.random.RandomState(seed)
    t = oracle.OracleTree(SIZE)
    t.frames[:] = np.frombuffer(rs.bytes(SIZE * oracle.FRAME), np.uint8).reshape(SIZE, oracle.FRAME)
    t.action[:] = rs.randint(0, 18, SIZE)
    t.reward[:] = rs.uniform(-2, 2, SIZE).astype(np.float32)
    pos = 0
    while pos < SIZE:
        L = min(int(rs.randint(5, 61)), SIZE - pos)
        t.timestep[pos:pos + L] = np.arange(L)
        t.nonterminal[pos:pos + L] = 1
        t.nonterminal[pos + L - 1] = 0
        pos += L
    return t


def cut_cases(H, n, seed):
    """(ring, sample indices, k each): for every k in 1 .. n - 1 a sample cut k steps on -- the last of them with its final
    observation on record 0, at the ring's wrap -- then, for n > 5, one window holding two short episodes that each end in
    a final observation (the first caps), and samples with no final observation in their window."""
    ring = base_ring(seed)
    rs = np.random.RandomState(seed + 1)
    stride = H + n + 4
    idxs, ks = [], []
    for k in range(1, n):
        idxs.append((H + 2 + (k - 1) * stride) % SIZE if k < n - 1 else SIZE - k)
        ks.append(k)
    pairs = list(zip(idxs, ks))
    if n > 5:   # two short episodes: F at idx + 2, then an episode of two records and F at idx + 5
        idx2 = SIZE - 300
        pairs += [(idx2, 2), (idx2 + 3, 2)]
        idxs.append(idx2)
        ks.append(2)
    used = set()
    for i, k in pairs:
        used |= {(i + j) % SIZE for j in range(-H - n, n + H + 1)}
    assert len(set((i + k) % SIZE for i, k in pairs)) == len(pairs)
    trunc_ref.final_ring(ring, [p[0] for p in pairs], [p[1] for p in pairs])
    free = [i for i in range(SIZE) if i not in used and trunc_ref.cut(ring, i, n) == n]
    uncut = list(rs.choice(free, min(6, len(free)), replace=False)) if free else []
    return ring, np.array(idxs + uncut, np.int64), np.array(ks + [n] * len(uncut), np.int64)


GRID = [(H, n) for H in (1, 4) for n in (1, 3, 20, 36)]


@pytest.mark.parametrize("H,n", GRID, ids=lambda v: str(v))
def test_trunc_ref_equals_the_fixed_horizon_gather_at_n_equals_k(H, n):
    ring, idx, want_k = cut_cases(H, n, 10 * H + n)
    gp = np.array([GAMMA ** j for j in range(64)], np.float32)
    gamma_n = np.float32(GAMMA ** n)
    s, a, r, ns, nt, k = trunc_ref.gather_trunc(ring, idx, H, n, gp[:n], gamma_n)
    assert_bits_equal(k, want_k, "cut offsets")
    assert set(range(1, n)) <= set(k.tolist())
    for kk in sorted(set(k.tolist())):
        rows = np.flatnonzero(k == kk)
        o = oracle.gather(ring, idx[rows], H, kk, gp[:kk])
        what = f"H {H}, n {n}, k {kk}"
        for got, want, name in ((s[rows], o[0], "states"), (a[rows], o[1], "actions"), (r[rows], o[2], "returns"),
                                (ns[rows], o[3], "next states")):
            assert_bits_equal(got, want, f"{what}: {name}")
        gamma_k = np.float32(GAMMA ** kk)
        assert_bits_equal(nt[rows], (o[4] * gamma_k).astype(np.float32), f"{what}: nonterminals")
        if kk < n:   # every cut sample bootstraps from its final observation
            assert (nt[rows] == gamma_k).all(), what


def test_two_short_episodes_in_one_window_are_cut_at_the_first():
    ring, idx, k = cut_cases(4, 20, 7)
    i = int(np.flatnonzero(idx == SIZE - 300)[0])
    assert k[i] == 2
    assert (ring.nonterminal[(idx[i] + np.arange(1, 20)) % SIZE] == trunc_ref.FINAL).sum() == 2
    assert trunc_ref.cut(ring, idx[i], 20) == 2


def test_final_at_the_wrap_is_record_zero():
    for n in (3, 20, 36):
        ring, idx, k = cut_cases(4, n, n)
        assert ((idx + k) % SIZE == 0).any() and ring.nonterminal[0] == trunc_ref.FINAL
