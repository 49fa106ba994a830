"""ReplayMemory.extend, host side: the new C entries' declarations against the ctypes bindings and their host refusals
(no launch is reached, so no GPU is needed), every refusal of extend() leaving the replay untouched, and
tests/extend_ref.py -- the timestep scan and the level-wise float32 tree rebuild -- bitwise against sequences of
oracle.OracleTree.append at capacities 1, 2, 13, 64 and 1000, every start head of a small ring, and k up to 3 cap + 2."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import extend_ref
import oracle
from helpers import assert_bits_equal

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RB_ERR_INVAL, RB_ERR_RANGE = -22, -34
FRAME = 84 * 84


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


# ---- the C entries -----------------------------------------------------------------------------------------------------------
_CT = {"float*": ctypes.c_void_p, "const float*": ctypes.c_void_p, "uint8_t*": ctypes.c_void_p,
       "const uint8_t*": ctypes.c_void_p, "int32_t*": ctypes.c_void_p, "const int32_t*": ctypes.c_void_p,
       "int64_t*": ctypes.c_void_p, "void*": ctypes.c_void_p, "int64_t": ctypes.c_int64, "rb_stream_t": ctypes.c_void_p}


def _header_decl(name):
    text = open(os.path.join(ROOT, "include", "rainbow_b200.h")).read()
    m = re.search(r"(\w+)\s+" + name + r"\s*\(([^)]*)\)", text)
    return m.group(1), m.group(2).split(",")


def test_signatures_match_the_header():
    from rainbow_b200 import _lib
    ret, decl = _header_decl("rb_append_bulk")
    types = [_CT[re.sub(r"\s*\w+$", "", a.strip()).replace(" *", "*")] for a in decl]
    names = [re.search(r"(\w+)$", a.strip()).group(1) for a in decl]
    assert ret == "int" and _lib.SIGNATURES["rb_append_bulk"] == (ctypes.c_int, types)
    assert names[10:] == ["head", "new_frames", "actions", "rewards", "flags", "k", "scratch", "scratch_bytes", "stream"]
    ret, decl = _header_decl("rb_append_bulk_scratch_bytes")
    assert ret == "int" and [a.strip() for a in decl] == ["int64_t k"]
    assert _lib.SIGNATURES["rb_append_bulk_scratch_bytes"] == (ctypes.c_int, [ctypes.c_int64])
    assert lib().rb_abi_version() == 3, "additive entries: the ABI version stays"


def test_scratch_bytes():
    f = lib().rb_append_bulk_scratch_bytes
    assert f(0) == 0 and f(-5) == 0
    assert f(1) == 8 and f(1024) == 8 and f(1025) == 12 and f(1 << 20) == 4 * (1024 + 1)


def _bulk(size=64, k=4, head=0, null=None, scratch_bytes=None):
    """rb_append_bulk with fake (never dereferenced) pointers: every case below is refused before any launch."""
    p = [0x1000 * (i + 1) for i in range(13)]
    if null is not None:
        p[null] = None
    tree, frames, ts, act, rew, nt, ring, rmax, new, a, r, f, scratch = p
    sb = lib().rb_append_bulk_scratch_bytes(k) if scratch_bytes is None else scratch_bytes
    return lib().rb_append_bulk(tree, extend_ref.tree_start(size), size, frames, ts, act, rew, nt, ring, rmax, head, new,
                                a, r, f, k, scratch, sb, None)


@pytest.mark.parametrize("null", range(13))
def test_entry_refuses_null_pointers(null):
    assert _bulk(null=null) == RB_ERR_INVAL


def test_entry_refusals():
    assert _bulk(size=63) == RB_ERR_INVAL
    assert _bulk(size=0) == RB_ERR_INVAL
    assert _bulk(k=0) == RB_ERR_RANGE and _bulk(k=65) == RB_ERR_RANGE and _bulk(k=-1) == RB_ERR_RANGE
    assert _bulk(head=-1) == RB_ERR_RANGE and _bulk(head=64) == RB_ERR_RANGE
    assert _bulk(k=2000, size=4096, scratch_bytes=8) == RB_ERR_RANGE
    assert b"scratch" in lib().rb_last_error()


# ---- extend()'s refusals ------------------------------------------------------------------------------------------------------
class _Ring:
    def __init__(self):
        self.index, self.full, self.size = 5, False, 64


def bare_memory(switch=False):
    """A ReplayMemory without device state: every refusal happens before the ring, the queue or the device is touched."""
    from rainbow_b200.memory import ReplayMemory
    mem = ReplayMemory.__new__(ReplayMemory)
    mem.bootstrap_truncation, mem.defer_appends, mem.t = switch, True, 7
    mem._queue = ["queued"]
    mem.transitions = _Ring()
    mem.device = torch.device("cuda", 0)
    return mem


def good(k=6):
    return (np.zeros((k, 84, 84), np.uint8), np.arange(k) % 4, np.ones(k, np.float32), np.zeros(k, bool))


def untouched(mem):
    assert mem._queue == ["queued"] and mem.t == 7
    assert (mem.transitions.index, mem.transitions.full) == (5, False)
    assert getattr(mem, "_bulk", None) is None


def _replace(i, v, k=6):
    args = list(good(k))
    args[i] = v
    return args


REFUSALS = {
    "frames rank": _replace(0, np.zeros((6, 84), np.uint8)),
    "frames shape": _replace(0, np.zeros((6, 84, 83), np.uint8)),
    "frames flat shape": _replace(0, np.zeros((6, 7057), np.uint8)),
    "frames int16": _replace(0, np.zeros((6, 84, 84), np.int16)),
    "frames float32": _replace(0, np.zeros((6, 84, 84), np.float32)),
    "frames float tensor": _replace(0, torch.zeros(6, 7056)),
    "actions length": _replace(1, np.zeros(5, np.int64)),
    "actions 2-d": _replace(1, np.zeros((6, 1), np.int64)),
    "actions float": _replace(1, np.zeros(6, np.float32)),
    "actions beyond int32": _replace(1, np.array([0, 1, 2, 3, 2 ** 31, 0])),
    "actions below int32": _replace(1, np.array([0, 1, 2, 3, -2 ** 31 - 1, 0])),
    "rewards length": _replace(2, np.zeros(7, np.float32)),
    "rewards strings": _replace(2, np.array(["a"] * 6)),
    "terminals length": _replace(3, np.zeros(4, bool)),
    "terminals float": _replace(3, np.zeros(6, np.float64)),
}


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_extend_refusals_leave_the_replay_untouched(case):
    mem = bare_memory()
    with pytest.raises(ValueError):
        mem.extend(*REFUSALS[case])
    untouched(mem)


def test_float_frames_name_the_quantisation():
    mem = bare_memory()
    with pytest.raises(ValueError, match=r"astype\(np.int32\).astype\(np.uint8\)"):
        mem.extend(*_replace(0, np.zeros((6, 84, 84), np.float32)))


def test_final_needs_the_switch():
    from rainbow_b200._lib import RainbowB200Error
    mem = bare_memory(False)
    with pytest.raises(RainbowB200Error, match="bootstrap_truncation"):
        mem.extend(*good(), final=np.zeros(6, bool))
    untouched(mem)


def _final_case(j=3, **edit):
    frames, a, r, term = good()
    a, r, term = a.copy(), r.copy(), term.copy()
    a[j], r[j] = 0, 0.0
    fin = np.zeros(6, bool)
    fin[j] = True
    for key, (pos, v) in edit.items():
        {"a": a, "r": r, "term": term, "fin": fin}[key][pos] = v
    return (frames, a, r, term), fin


FINAL_REFUSALS = {
    "at j = 0": ((0,), {}),
    "after a terminal": ((3,), dict(term=(2, True))),
    "after another final": ((3,), dict(fin=(2, True), a=(2, 0), r=(2, 0.0))),
    "itself terminal": ((3,), dict(term=(3, True))),
    "nonzero action": ((3,), dict(a=(3, 2))),
    "nonzero reward": ((3,), dict(r=(3, 0.5))),
    "negative zero reward": ((3,), dict(r=(3, -0.0))),
}


@pytest.mark.parametrize("case", sorted(FINAL_REFUSALS))
def test_final_refusals_leave_the_replay_untouched(case):
    (j,), edit = FINAL_REFUSALS[case]
    args, fin = _final_case(j, **edit)
    mem = bare_memory(True)
    with pytest.raises(ValueError, match="final record"):
        mem.extend(*args, final=fin)
    untouched(mem)
    with pytest.raises(ValueError):
        mem.extend(*args, final=fin[:5])
    untouched(mem)


def test_accepted_final_pattern_converts_to_flags():
    args, fin = _final_case(3)
    mem = bare_memory(True)
    fr, acts, rews, flags = mem._check_extend(*args, fin)
    assert list(flags) == [0, 0, 0, 2, 0, 0] and fr.shape == (6, FRAME) and fr.dtype == torch.uint8
    assert acts.dtype == np.int32 and rews.dtype == np.float32


def test_rewards_round_as_append_rounds():
    """append passes float(reward) through ctypes' c_float: round to nearest from the double."""
    mem = bare_memory()
    r = np.array([0.1, 1e-46, 3.4028235e38, 1 + 2 ** -24 + 2 ** -60, 2 ** 60 + 1, -7], dtype=object)
    for rewards in (r.astype(np.float64), np.array([1, 2 ** 40 + 1, -3, 2 ** 53 + 1, 0, 5], np.int64)):
        _, _, rews, _ = mem._check_extend(np.zeros((6, FRAME), np.uint8), np.zeros(6, np.int64), rewards, np.zeros(6, bool),
                                          None)
        want = np.array([ctypes.c_float(float(x)).value for x in rewards], np.float32)
        assert_bits_equal(rews, want, "rewards")


# ---- the reference against the oracle's appends ------------------------------------------------------------------------------
def oracle_tree(size):
    """OracleTree whose sum tree has one zero past its end: an odd size's last leaf reads a right sibling there."""
    ot = oracle.OracleTree(size)
    n = ot.sum_tree.size
    ot.sum_tree = np.zeros(n + 1, np.float32)[:n]
    return ot


def random_ring(size, head, rs, t0):
    ot = oracle_tree(size)
    leaves = np.arange(size) + ot.tree_start
    ot.update(leaves, rs.uniform(0.01, 3.0, size).astype(np.float32))   # siblings are not all the running max
    ot.max[0] = np.float32(rs.uniform(3.0, 5.0))
    ot.index, ot.full = head, bool(rs.randint(2))
    return ot, t0


def ring_of(ot, t):
    return dict(size=ot.size, tree=ot.sum_tree.copy(), timestep=ot.timestep.copy(), action=ot.action.copy(),
                reward=ot.reward.copy(), nonterminal=ot.nonterminal.copy(), index=ot.index, full=ot.full, t=t,
                max=ot.max[0])


def records(k, rs, pattern, with_final):
    a = rs.randint(0, 18, k).astype(np.int32)
    r = rs.choice(np.array([-1, 0, 1, 0.5, 2.25], np.float32), k)
    term = {"none": np.zeros(k, bool), "all": np.ones(k, bool), "random": rs.uniform(size=k) < 0.2,
            "last": np.arange(k) == k - 1}[pattern]
    flags = term.astype(np.uint8)
    if with_final:
        for j in range(1, k):
            if flags[j - 1] == 0 and rs.uniform() < 0.15:
                flags[j] = extend_ref.FINAL
                a[j], r[j] = 0, 0.0
    return a, r, flags


def appended(ot, t, a, r, flags):
    """The same records through OracleTree.append one by one (append_truncated's pair for a final observation)."""
    for j in range(len(flags)):
        fin = flags[j] == extend_ref.FINAL
        slot = ot.index
        ot.append(t, np.zeros(FRAME, np.uint8), int(a[j]), np.float32(r[j]), flags[j] == 0,
                  value=0.0 if fin else None)
        if fin:
            ot.nonterminal[slot] = extend_ref.FINAL
        t = 0 if flags[j] else t + 1
    return t


def assert_ring_equal(got, ot, t):
    assert_bits_equal(got["tree"], ot.sum_tree, "tree")
    for key in ("timestep", "action", "reward", "nonterminal"):
        assert_bits_equal(got[key], getattr(ot, key), key)
    assert (got["index"], got["full"], got["t"]) == (ot.index, ot.full, t)


@pytest.mark.parametrize("size", [1, 2, 13, 64, 1000])
@pytest.mark.parametrize("pattern", ["none", "all", "random", "last"])
def test_reference_equals_sequential_appends(size, pattern):
    rs = np.random.RandomState(size * 7 + len(pattern))
    ks = sorted({1, 2, 7, 8, 9, max(1, size - 1), size, size + 5, 3 * size + 2})
    heads = range(size) if size <= 13 else (0, size // 2, size - 1)
    for head in heads:
        for k in ks:
            for with_final in (False, True):
                ot, t0 = random_ring(size, head, rs, int(rs.randint(0, 50)))
                a, r, flags = records(k, rs, pattern, with_final)
                got = extend_ref.extend(ring_of(ot, t0), a, r, flags)
                t = appended(ot, t0, a, r, flags)
                assert_ring_equal(got, ot, t)


def test_timesteps_scan():
    t, t_end = extend_ref.timesteps(np.array([0, 0, 1, 0, 2, 0, 0, 1], np.uint8), 5)
    assert list(t) == [5, 6, 7, 0, 1, 0, 1, 2] and t_end == 0
    t, t_end = extend_ref.timesteps(np.zeros(3, np.uint8), 9)
    assert list(t) == [9, 10, 11] and t_end == 12
