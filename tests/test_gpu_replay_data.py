"""The replay's data path against the CPU oracle (oracle/rb_oracle.c), bitwise: rb_gather (k_gather), rb_gather_horizon
without augmentation (k_gather_hz), rb_iter_states (k_iter_states) with the Python iterator and evaluate_q_memory's
chunks, and rb_append / rb_append_batch (k_append_batch).

Every value on this path is exact -- a byte divided by 255, a fp32 sum in a fixed order, integer bookkeeping -- so every
comparison is bitwise.  Each case prefills its outputs with NaN (-7 for int64), keeps two guard rows past the last one
the kernel may write, replays the launch from a CUDA graph into a second set of outputs, and checks refused calls write
nothing.  The rings the gathers read sit inside device buffers with 64 records of junk on either side, so an index the
kernels fail to wrap reads junk (and fails the comparison) instead of memory outside the allocation.  The host checks at
the top assert the case tables reach every window slot position with an episode start, windows without one and with
several, both ends of the ring, and both of the gather's CTA splits."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from helpers import assert_bits_equal

DEV = "cuda:0"
FRAME = 84 * 84
MARGIN = 64               # junk records before and after every ring array the gathers and the iterator read
SM_COUNT = 132            # rbi::SM_COUNT; gather_grid splits each window slot in two while used slots * B < 2 * SM_COUNT
RB_ERR_INVAL, RB_ERR_RANGE = -22, -34
RING = 512                # records of the ring the gathers and the iterator read


# ---- rings with designed episodes (host) --------------------------------------------------------------------------------
def ring_timesteps(size, long_len, rs):
    """Episodes laid out around the ring: first one of long_len records that ends at record 9 (so it spans the ring's
    wrap), then episodes of 1, 1, 2, 1, 3, 1, 4 records, then of 1 to 4 records with one of 70 about every 17 episodes."""
    lengths = [long_len, 1, 1, 2, 1, 3, 1, 4]
    left = size - sum(lengths)
    while left > 0:
        n = 70 if rs.uniform() < 0.06 else int(rs.randint(1, 5))
        lengths.append(min(n, left))
        left -= lengths[-1]
    ts = np.empty(size, np.int32)
    last = np.zeros(size, bool)
    pos = size - long_len + 10
    for n in lengths:
        for k in range(n):
            ts[(pos + k) % size] = k
        last[(pos + n - 1) % size] = True
        pos += n
    return ts, last


def host_ring(size, seed, long_len=100):
    """An OracleTree holding random frame bytes, non-integer fp32 rewards, actions, the episodes of ring_timesteps and
    nonterminal 0 at the last record of each episode."""
    rs = np.random.RandomState(seed)
    t = oracle.OracleTree(size)
    ts, last = ring_timesteps(size, long_len, rs)
    t.timestep[:] = ts
    t.nonterminal[:] = ~last
    t.frames[:] = np.frombuffer(rs.bytes(size * FRAME), np.uint8).reshape(size, FRAME)
    t.action[:] = rs.randint(0, 18, size)
    t.reward[:] = rs.uniform(-2, 2, size).astype(np.float32)
    return t


def window_firsts(t, idx, start, W):
    """[len(idx), W] bool: window slot s of sample i (record idx_i - start + s, wrapped) starts an episode."""
    rec = (np.asarray(idx)[:, None] - start + np.arange(W)) % t.size
    return t.timestep[rec] == 0


def coverage_rows(t, start, W, rs):
    """Indices whose windows (W records from idx - start) have: no episode start; several; a start at slot p, for each p."""
    f = window_firsts(t, np.arange(t.size), start, W)
    none = rs.choice(np.flatnonzero(~f.any(1)))
    several = rs.choice(np.flatnonzero(f.sum(1) >= 2))
    return none, several, [int(rs.choice(np.flatnonzero(f[:, p]))) for p in range(W)]


def gather_split(H, n, B):
    used = H + n if H + n < 2 * H else 2 * H
    return 2 if used * B < 2 * SM_COUNT else 1


# ---- the gather's case table --------------------------------------------------------------------------------------------
def gather_pairs():
    """(history, n): n = 1, n < history, n = history, n > history, and history + n = 32, 33, 64, for history 1 ... 8, 16,
    32; windows up to RB_MAX_WINDOW = 64."""
    out = []
    for H in (1, 2, 3, 4, 5, 6, 7, 8, 16, 32):
        ns = {1, H, H + 1, 32 - H, 33 - H, 64 - H}
        if H > 2:
            ns.add((H + 1) // 2)
        out += [(H, n) for n in sorted(ns) if n >= 1 and H + n <= 64]
    return out


def gather_cases():
    """(H, n, B, slot offset, seed): per (H, n) one case of B 96 (64 at a 64-record window, plus B 31 for the slot positions
    that leaves out) and one of B 1, 31, 37 or 38; and B 512 / 2048 at a few small windows."""
    cases = []
    small = (1, 31, 37, 38)
    for i, (H, n) in enumerate(gather_pairs()):
        W = H + n
        if W < 64:
            cases.append((H, n, 96, 0, i))
        else:
            cases += [(H, n, 64, 0, i), (H, n, 31, 57, 1000 + i)]
        cases.append((H, n, small[i % 4], (7 * i) % W, 2000 + i))
    cases += [(4, 3, 37, 0, 3000), (4, 3, 38, 0, 3001), (4, 3, 512, 0, 3002), (4, 3, 2048, 0, 3003), (1, 3, 512, 0, 3004),
              (8, 8, 512, 0, 3005), (2, 1, 2048, 0, 3006)]
    return cases


def gather_indices(t, H, n, B, off, seed):
    """0, 1, size - 1, the last index whose window wraps at the start and the first that wraps at the end, a window without
    an episode start, one with several, then windows with a start at slot (off + j) mod W; the rest random."""
    rs = np.random.RandomState(seed)
    W, size = H + n, t.size
    none, several, at_slot = coverage_rows(t, H - 1, W, rs)
    rows = [0, 1, size - 1, (H - 2) % size, size - n, none, several]
    rows += [at_slot[(off + j) % W] for j in range(W)]
    rows += list(rs.randint(0, size, max(0, B - len(rows))))
    return np.array(rows[:B], np.int64)


def case_id(c):
    H, n, B, off, seed = c
    return f"h{H}-n{n}-b{B}-split{gather_split(H, n, B)}" + (f"-off{off}" if off else "")


def iter_cases():
    """(history, first, count): history 1 ... 8 and 64 at first 0, size - 1 and size - history + 1, count 1, 64 and 65."""
    return [(H, first, count) for H in (1, 2, 3, 4, 5, 6, 7, 8, 64)
            for first in sorted({0, RING - 1, RING - H + 1}) for count in (1, 64, 65)]


def test_case_tables_cover_the_windows():
    """Host check of the tables above: for every (history, n) of the gather an episode start at every window slot, a
    window with none and one with several, indices 0, 1 and size - 1, windows across both ends of the ring; both splits
    and every batch size; the same episode-start coverage for every history of the iterator."""
    t = host_ring(RING, 0)
    seen = {}
    for c in gather_cases():
        H, n, B, off, seed = c
        assert H + n <= 64 and (H + n < 64 or B <= 64)
        idx = gather_indices(t, H, n, B, off, seed)
        f = window_firsts(t, idx, H - 1, H + n)
        s = seen.setdefault((H, n), dict(slots=set(), none=False, several=False, idx=set(), wrap0=False, wrap1=False))
        s["slots"] |= set(np.flatnonzero(f.any(0)))
        s["none"] |= bool((~f.any(1)).any())
        s["several"] |= bool((f.sum(1) >= 2).any())
        s["idx"] |= set(idx.tolist())
        s["wrap0"] |= bool((idx < H - 1).any())
        s["wrap1"] |= bool((idx + n >= RING).any())
    assert set(gather_pairs()) <= set(seen)
    for (H, n), s in seen.items():
        assert s["slots"] == set(range(H + n)), (H, n, set(range(H + n)) - s["slots"])
        assert s["none"] and s["several"] and {0, 1, RING - 1} <= s["idx"], (H, n)
        assert s["wrap1"] and (s["wrap0"] or H == 1), (H, n)
    assert {gather_split(H, n, B) for H, n, B, _, _ in gather_cases()} == {1, 2}
    assert {1, 31, 37, 38, 512, 2048} <= {c[2] for c in gather_cases()}
    assert {64 - H for H in (1, 2, 3, 4, 5, 6, 7, 8, 16, 32)} <= {n for H, n in gather_pairs() if H + n == 64}
    for H in (1, 2, 3, 4, 5, 6, 7, 8, 64):
        cur = np.concatenate([first + np.arange(count) for h, first, count in iter_cases() if h == H])
        f = window_firsts(t, cur, H - 1, H)
        assert set(np.flatnonzero(f.any(0))) == set(range(H)), H
        assert (~f[:, 1:].any(1)).any() and (H < 3 or (f[:, 1:].sum(1) >= 2).any()), H


# ---- device side ---------------------------------------------------------------------------------------------------------
def lib():
    from rainbow_b200 import _lib
    return _lib.load()


def p(x):
    return None if x is None else x.data_ptr()


def cpu(x):
    return x.detach().cpu().numpy()


def stream():
    return torch.cuda.current_stream().cuda_stream


def padded(a, junk):
    """a on the device inside junk records on either side; returns (whole buffer, view of a)."""
    whole = torch.from_numpy(np.concatenate([junk, a, junk])).to(DEV)
    return whole, whole[MARGIN:MARGIN + a.shape[0]]


class DeviceRing:
    """The arrays of a host ring on the device, each inside MARGIN junk records on either side."""

    def __init__(self, t, seed=99):
        rs = np.random.RandomState(seed)
        self.size = t.size
        self._keep = []
        for name, junk in (("frames", np.frombuffer(rs.bytes(MARGIN * FRAME), np.uint8).reshape(MARGIN, FRAME)),
                           ("timestep", rs.choice(np.array([0, 7], np.int32), MARGIN)),
                           ("action", np.full(MARGIN, 99, np.int32)),
                           ("reward", np.full(MARGIN, 1000.0, np.float32)),
                           ("nonterminal", rs.randint(0, 2, MARGIN).astype(np.uint8))):
            whole, view = padded(getattr(t, name), junk)
            self._keep.append(whole)
            setattr(self, name, view)
        assert self.frames.data_ptr() % 16 == 0


class GatherOut:
    """Output buffers with two guard rows past B: NaN, and -7 for the int64 actions."""

    def __init__(self, B, H):
        self.B, self.H = B, H
        self.states = torch.full((B + 2, H, 84, 84), float("nan"), device=DEV)
        self.next_states = torch.full((B + 2, H, 84, 84), float("nan"), device=DEV)
        self.actions = torch.full((B + 2,), -7, dtype=torch.int64, device=DEV)
        self.returns = torch.full((B + 2,), float("nan"), device=DEV)
        self.nonterminals = torch.full((B + 2,), float("nan"), device=DEV)

    def tensors(self):
        return self.states, self.next_states, self.actions, self.returns, self.nonterminals

    def assert_guards(self, what):
        B = self.B
        for x in self.tensors():
            g = x[B:]
            ok = (g == -7).all() if x.dtype == torch.int64 else torch.isnan(g).all()
            assert bool(ok), f"{what}: a guard row past B was written"

    def assert_untouched(self, what):
        for x in self.tensors():
            ok = (x == -7).all() if x.dtype == torch.int64 else torch.isnan(x).all()
            assert bool(ok), f"{what}: a refused call wrote its outputs"

    def assert_same(self, other, what):
        for a, b in zip(self.tensors(), other.tensors()):
            assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                               b.view(torch.int32) if b.dtype == torch.float32 else b), what


def gather_args(ring, didx, H, n, window, out):
    return (p(ring.frames), p(ring.timestep), p(ring.action), p(ring.reward), p(ring.nonterminal), ring.size, p(didx),
            out.B, H, n, p(window), p(out.states), p(out.next_states), p(out.actions), p(out.returns), p(out.nonterminals))


def eager_and_graph(launch, B, H):
    """Runs launch(out) eagerly into one output set and as a CUDA-graph replay into another; both must agree bitwise."""
    eager, replay = GatherOut(B, H), GatherOut(B, H)
    assert launch(eager) == 0, lib().rb_last_error()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            rc = launch(replay)
    torch.cuda.current_stream().wait_stream(s)
    assert rc == 0, lib().rb_last_error()
    g.replay()
    torch.cuda.synchronize()
    eager.assert_guards("eager")
    replay.assert_guards("graph replay")
    eager.assert_same(replay, "graph replay differs from the eager launch")
    return eager


def assert_gather_equals_oracle(out, ref, what):
    B = out.B
    s, a, r, ns, nt = ref
    assert_bits_equal(cpu(out.states[:B]), s, f"{what}: states")
    assert_bits_equal(cpu(out.next_states[:B]), ns, f"{what}: next states")
    assert_bits_equal(cpu(out.actions[:B]), a, f"{what}: actions")
    assert_bits_equal(cpu(out.returns[:B]), r, f"{what}: returns")
    return cpu(out.nonterminals[:B]), nt.reshape(-1)


@pytest.fixture(scope="module")
def rings():
    t = host_ring(RING, 0)
    return t, DeviceRing(t)


# ---- rb_gather -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", gather_cases(), ids=case_id)
def test_gather_equals_oracle(rings, case):
    t, ring = rings
    H, n, B, off, seed = case
    idx = gather_indices(t, H, n, B, off, seed)
    didx = torch.from_numpy(idx).to(DEV)
    gp_host = np.array([0.99 ** k for k in range(n)], np.float32)
    gp = torch.from_numpy(gp_host).to(DEV)
    out = eager_and_graph(lambda o: lib().rb_gather(*gather_args(ring, didx, H, n, gp, o), stream()), B, H)
    got_nt, want_nt = assert_gather_equals_oracle(out, oracle.gather(t, idx, H, n, gp_host), case_id(case))
    assert_bits_equal(got_nt, want_nt, "nonterminals")


@pytest.mark.gpu
def test_gather_refusals_write_nothing(rings):
    """A window of 65 records, a batch past 65535, or non-positive sizes are refused with their code and write nothing."""
    _, ring = rings
    didx = torch.zeros(4, dtype=torch.int64, device=DEV)
    gp = torch.ones(64, device=DEV)
    for H, n, code in ((32, 33, RB_ERR_RANGE), (1, 64, RB_ERR_RANGE), (16, 49, RB_ERR_RANGE), (64, 1, RB_ERR_RANGE),
                       (0, 3, RB_ERR_INVAL), (4, 0, RB_ERR_INVAL)):
        out = GatherOut(4, max(H, 1))
        assert lib().rb_gather(*gather_args(ring, didx, H, n, gp, out), stream()) == code, (H, n)
        torch.cuda.synchronize()
        out.assert_untouched(f"history {H}, n {n}")


# ---- rb_gather_horizon, no augmentation ----------------------------------------------------------------------------------
def horizon_row(n, n_t, g):
    """An rb_horizon row on the device whose n field is n and whose powers are those of n_t ... 64 with discount g."""
    from rainbow_b200.horizon import ROW_DTYPE
    r = np.zeros(1, dtype=ROW_DTYPE)
    r["n"], r["gamma_n"] = n, np.float32(g ** n_t)
    r["gamma_pow"][0] = np.array([g ** k for k in range(64)]).astype(np.float32)
    return torch.from_numpy(r.view(np.uint8).copy()).to(DEV), r["gamma_pow"][0].copy(), np.float32(g ** n_t)


@pytest.mark.gpu
@pytest.mark.parametrize("H,n_max,B", [(4, 3, 37), (4, 10, 96), (1, 5, 31), (8, 12, 300), (16, 20, 64)],
                         ids=lambda v: str(v))
def test_gather_horizon_equals_oracle_at_every_n(rings, H, n_max, B):
    """k_gather_hz at the row's n_t for n_t = 1 ... n_max: the oracle's gather at n = n_t, with the nonterminals in discount
    form fl32(nt * gamma_n).  A row n of 0 or -3 gathers at n_t = 1, one above n_max at n_t = n_max."""
    t, ring = rings
    idx = gather_indices(t, H, n_max, B, 0, 11 * H + n_max)
    didx = torch.from_numpy(idx).to(DEV)
    rows = [(n, n) for n in range(1, n_max + 1)] + [(0, 1), (-3, 1), (n_max + 1, n_max), (n_max + 3, n_max)]
    for n_row, n_t in rows:
        row, gp_host, gamma_n = horizon_row(n_row, n_t, 0.97)
        out = eager_and_graph(lambda o: lib().rb_gather_horizon(*gather_args(ring, didx, H, n_max, row, o), 0, 0.0, 1, 1,
                                                                0, None, None, None, stream()), B, H)
        got_nt, want_nt = assert_gather_equals_oracle(out, oracle.gather(t, idx, H, n_t, gp_host[:n_t]),
                                                      f"row n {n_row}, n_t {n_t}")
        assert_bits_equal(got_nt, (want_nt * gamma_n).astype(np.float32), f"nonterminals, n_t {n_t}")


# ---- rb_iter_states and the Python iterator ------------------------------------------------------------------------------
def iter_launch(ring, first, count, H, out):
    return lib().rb_iter_states(p(ring.frames), p(ring.timestep), ring.size, first, count, H, p(out), stream())


@pytest.mark.gpu
@pytest.mark.parametrize("H", [1, 2, 3, 4, 5, 6, 7, 8, 64])
def test_iter_states_equal_oracle(rings, H):
    t, ring = rings
    for h, first, count in iter_cases():
        if h != H:
            continue
        outs = []
        for replay in (False, True):
            out = torch.full((count + 2, H, 84, 84), float("nan"), device=DEV)
            if replay:
                g = torch.cuda.CUDAGraph()
                s = torch.cuda.Stream()
                s.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(s):
                    with torch.cuda.graph(g, stream=s):
                        rc = iter_launch(ring, first, count, H, out)
                torch.cuda.current_stream().wait_stream(s)
                g.replay()
            else:
                rc = iter_launch(ring, first, count, H, out)
            assert rc == 0, lib().rb_last_error()
            torch.cuda.synchronize()
            assert bool(torch.isnan(out[count:]).all()), "guard rows written"
            outs.append(out)
        assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), "graph replay differs"
        want = np.stack([oracle.iter_state(t, first + j, H) for j in range(count)])
        assert_bits_equal(cpu(outs[0][:count]), want, f"first {first}, count {count}")


@pytest.mark.gpu
def test_iter_states_full_grid_and_refusals(rings):
    """count = 65535 (the grid's y limit) at history 1: the first ring's worth of states against the oracle, the rest
    equal to the state one ring earlier.  count 65536, count 0, history 65 and history 0 are refused and write nothing."""
    t, ring = rings
    count, first = 65535, RING - 1
    out = torch.full((count + 2, 1, 84, 84), float("nan"), device=DEV)
    assert iter_launch(ring, first, count, 1, out) == 0, lib().rb_last_error()
    torch.cuda.synchronize()
    assert bool(torch.isnan(out[count:]).all())
    want = np.stack([oracle.iter_state(t, first + j, 1) for j in range(RING)])
    assert_bits_equal(cpu(out[:RING]), want, "first ring of states")
    assert torch.equal(out[RING:count].view(torch.int32), out[:count - RING].view(torch.int32)), "period of the ring"
    del out
    small = torch.full((4, 64, 84, 84), float("nan"), device=DEV)
    for cnt, H in ((65536, 1), (0, 1), (1, 65), (1, 0), (-1, 1)):
        assert iter_launch(ring, 0, cnt, H, small) == RB_ERR_RANGE, (cnt, H)
    torch.cuda.synchronize()
    assert bool(torch.isnan(small).all())


def make_args(**kw):
    import argparse
    d = dict(device=torch.device(DEV), history_length=4, discount=0.99, multi_step=3, priority_weight=0.4,
             priority_exponent=0.5)
    d.update(kw)
    return argparse.Namespace(**d)


@pytest.mark.gpu
@pytest.mark.parametrize("H", [1, 4])
def test_python_iterator_and_evaluate_q_memory_chunks(H):
    """iter(ReplayMemory) at capacity 130 (not a multiple of its 64-state chunks) yields the oracle's iterator states up to
    StopIteration, and evaluate_q_memory's chunks (64 and 50) pass the same states to the network."""
    from rainbow_b200.agent import Agent
    from rainbow_b200.memory import ReplayMemory
    cap = 130
    t = host_ring(cap, 5, long_len=40)
    mem = ReplayMemory(make_args(history_length=H), cap, seed=0)
    mem.transitions.load_arrays(frames=t.frames, timestep=t.timestep, action=t.action, reward=t.reward,
                                nonterminal=t.nonterminal, index=17, full=True)
    want = np.stack([oracle.iter_state(t, c, H) for c in range(cap)])
    got = np.stack([cpu(s) for s in mem])
    assert_bits_equal(got, want, "iter(memory)")
    with pytest.raises(StopIteration):
        next(mem)

    class Net:
        seen = []

        def q_select(self, states):
            self.seen.append(states.clone())
            return None, torch.zeros(states.shape[0], device=DEV)

    for chunk in (64, 50):
        net = Net()
        net.seen = []
        assert len(Agent.evaluate_q_memory(net, mem, chunk=chunk)) == cap
        assert [x.shape[0] for x in net.seen] == [min(chunk, cap - f) for f in range(0, cap, chunk)]
        assert_bits_equal(cpu(torch.cat(net.seen)), want, f"evaluate_q_memory, chunk {chunk}")


# ---- rb_append / rb_append_batch -----------------------------------------------------------------------------------------
def edge_frames(k, rs):
    """k float32 frames holding every quantisation edge -- 0, 1, each j / 255 and its fp32 neighbours, values in
    (0, 1/255) -- in a different order each, the rest uniform in [0, 1)."""
    q = np.arange(256, dtype=np.float32) / np.float32(255)
    edges = np.concatenate([q, np.nextafter(q, np.float32(0)), np.nextafter(q, np.float32(1)), [0.0, 1.0],
                            rs.uniform(0, 1 / 255, 200)]).astype(np.float32)
    edges = edges[(edges >= 0) & (edges <= 1)]
    out = rs.uniform(0, 1, (k, FRAME)).astype(np.float32)
    for j in range(k):
        out[j, rs.choice(FRAME, edges.size, replace=False)] = edges
    return out


class AppendCase:
    """A device SegmentTree and its OracleTree mirror holding random frames, records and leaves and a running max that is
    not 1; appends go to both, the in-episode step and the count of appends are tracked beside them."""

    def __init__(self, size, seed):
        from rainbow_b200.memory import SegmentTree
        rs = self.rs = np.random.RandomState(seed)
        self.ref = r = oracle.OracleTree(size)
        r.frames[:] = np.frombuffer(rs.bytes(size * FRAME), np.uint8).reshape(size, FRAME)
        r.timestep[:] = rs.randint(0, 50, size)
        r.action[:] = rs.randint(0, 18, size)
        r.reward[:] = rs.uniform(-1, 1, size).astype(np.float32)
        r.nonterminal[:] = rs.uniform(size=size) > 0.3
        r.update(np.arange(size) + r.tree_start, rs.uniform(0.01, 3, size).astype(np.float32))
        r.max[0] = np.float32(rs.uniform(0.5, 4))
        self.t_ep, self.count = int(rs.randint(0, 9)), 0
        self.dev = d = SegmentTree(size, DEV)
        d.load_arrays(sum_tree=r.sum_tree, frames=r.frames, timestep=r.timestep, action=r.action, reward=r.reward,
                      nonterminal=r.nonterminal, index=0, full=False, t_episode=self.t_ep, max_value=float(r.max[0]))

    def place_head(self, head):
        """Move the write head (and clear `full`) on both sides, keeping the in-episode step and the count."""
        self.ref.index, self.ref.full = head, False
        self.dev.ring_state[0], self.dev.ring_state[1] = head, 0

    def args(self, size=None):
        d = self.dev
        return (p(d.tree), d.tree_start, d.size if size is None else size, p(d.frames), p(d.timestep), p(d.action),
                p(d.reward), p(d.nonterminal), p(d.ring_state), p(d.running_max))

    def launch(self, frames, actions, rewards, terminals, single=False, size=None, frame_offset=0, k=None):
        k = len(actions) if k is None else k
        if single:
            return lib().rb_append(*self.args(size), frames[0].data_ptr() + frame_offset, int(actions[0]),
                                   float(rewards[0]), int(terminals[0]), stream())
        ptrs = (C.c_void_p * k)(*[frames[j % len(frames)].data_ptr() + frame_offset for j in range(k)])
        return lib().rb_append_batch(*self.args(size), ptrs, (C.c_int32 * k)(*[int(actions[j % len(actions)]) for j in range(k)]),
                                     (C.c_float * k)(*[float(rewards[j % len(rewards)]) for j in range(k)]),
                                     (C.c_int32 * k)(*[int(terminals[j % len(terminals)]) for j in range(k)]), k, stream())

    def oracle_append(self, frames_host, actions, rewards, terminals):
        for j in range(len(actions)):
            self.ref.append(self.t_ep, oracle.quantise_frame(frames_host[j]), int(actions[j]), np.float32(rewards[j]),
                            not terminals[j])
            self.t_ep = 0 if terminals[j] else self.t_ep + 1
            self.count += 1

    def assert_equal(self, what, frame_rows=None):
        torch.cuda.synchronize()
        d, r = self.dev, self.ref
        assert list(cpu(d.ring_state)) == [r.index, int(r.full), self.t_ep, self.count, 0], what
        assert_bits_equal(cpu(d.tree), r.sum_tree, f"{what}: tree")
        assert_bits_equal(cpu(d.running_max), r.max, f"{what}: running max")
        for name in ("timestep", "action", "reward", "nonterminal"):
            assert_bits_equal(cpu(getattr(d, name)), getattr(r, name), f"{what}: {name}")
        if frame_rows is None:
            assert_bits_equal(cpu(d.frames), r.frames, f"{what}: frames")
        else:
            rows = torch.from_numpy(np.asarray(frame_rows, np.int64)).to(DEV)
            assert_bits_equal(cpu(d.frames[rows]), r.frames[frame_rows], f"{what}: frames")


def append_frames(host, source):
    t = torch.from_numpy(host)
    t = t.pin_memory() if source == "pinned" else t.to(DEV)
    return [t[j] for j in range(host.shape[0])]


@pytest.mark.gpu
@pytest.mark.parametrize("source", ["device", "pinned"])
@pytest.mark.parametrize("size", [8, 1026, 65538])   # tree depths 3, 11, 17
def test_append_equals_oracle(size, source):
    """k = 1 ... 8 with the head placed so that the batch wraps after every lane (and once mid-ring), a terminal at every
    lane position (and none), the in-episode step carried from launch to launch, `full` set exactly when the head wraps;
    k = 1 alternates between rb_append and rb_append_batch."""
    c = AppendCase(size, seed=size)
    small = size <= 1026
    for k in range(1, 9):
        for j, head in enumerate([size - w for w in range(1, k + 1)] + [size // 2 - 1]):
            c.place_head(head)
            frames = edge_frames(k, c.rs)
            actions = c.rs.randint(0, 18, k)
            rewards = c.rs.uniform(-3, 3, k).astype(np.float32)
            terminals = np.arange(k) == j
            wrapped = head + k >= size
            src = append_frames(frames, source)   # alive until the launch has been waited for
            assert c.launch(src, actions, rewards, terminals, single=(k == 1 and j % 2 == 0)) == 0, lib().rb_last_error()
            c.oracle_append(frames, actions, rewards, terminals)
            assert c.ref.full == wrapped
            c.assert_equal(f"k {k}, head {head}", None if small else [(head + i) % size for i in range(k)] + [0, size - 1])
    c.assert_equal("after every launch")


@pytest.mark.gpu
def test_append_graph_replay_equals_eager():
    """A wrapping batch of 5 captured once and replayed twice leaves the ring, tree and ring_state the two eager launches
    leave."""
    a, b = AppendCase(1026, 7), AppendCase(1026, 7)
    a.place_head(1023)
    b.place_head(1023)
    host = edge_frames(5, np.random.RandomState(3))
    frames = append_frames(host, "device")
    acts, rews, terms = [1, 2, 3, 4, 5], np.float32([0.5, -0.25, 1.75, 3.0, -2.5]), [0, 1, 0, 0, 1]
    for _ in range(2):
        assert a.launch(frames, acts, rews, terms) == 0
        a.oracle_append(host, acts, rews, terms)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            assert b.launch(frames, acts, rews, terms) == 0
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    g.replay()
    a.assert_equal("eager")
    for name in ("tree", "frames", "timestep", "action", "reward", "nonterminal", "ring_state", "running_max"):
        assert torch.equal(getattr(a.dev, name), getattr(b.dev, name)), name


@pytest.mark.gpu
def test_append_refusals_write_nothing():
    """An odd size, a frame not 16-byte aligned, k = 9, and k = 4 into a ring of 2 are refused with their code."""
    c = AppendCase(8, 1)
    c.place_head(6)
    host = edge_frames(9, c.rs)
    frames = append_frames(host, "device")
    acts, rews, terms = list(range(9)), [0.5] * 9, [0] * 9
    assert c.launch(frames, acts[:3], rews, terms, size=7) == RB_ERR_INVAL
    assert c.launch(frames, acts[:1], rews, terms, size=7, single=True) == RB_ERR_INVAL
    assert c.launch(frames, acts[:3], rews, terms, frame_offset=4) == RB_ERR_INVAL
    assert c.launch(frames, acts[:1], rews, terms, frame_offset=4, single=True) == RB_ERR_INVAL
    assert c.launch(frames, acts, rews, terms, k=9) == RB_ERR_RANGE
    c.assert_equal("refused calls")
    two = AppendCase(2, 2)
    assert two.launch(frames, acts[:4], rews, terms) == RB_ERR_RANGE
    two.assert_equal("k > size")
