"""ReplayMemory.extend on the H100 (rb_append_bulk, DESIGN §23): the same transitions through extend() and through
append() / append_truncated() leave every array and host mirror of the replay bitwise equal -- at capacities 14, 64 and
1000 (the ring needs an even size, so 14 stands for 13), k across the ring's size and the launch batch, heads at 0,
mid-ring and one before the wrap, terminal patterns, final observations, pageable / pinned / CUDA frames, a staging chunk
small enough to split the fill (with a chunk boundary at the wrap), a non-empty defer queue and priorities written
beforehand.  Then a full-size fill of a 1M ring against tests/extend_ref.py and load_arrays, and an offline CQL run."""
import numpy as np
import pytest
import torch

import extend_ref
from helpers import assert_bits_equal
from test_gpu_parity import DEV, FakeEnv, cpu, make_args

pytestmark = pytest.mark.gpu

FRAME = 84 * 84
POOL = 32


def frames_for(q):
    """Float frames in [0, 1] whose append quantisation (uint8)(int)fl32(f * 255) is q: f = fl32((q + 0.5) / 255)."""
    f = ((q.astype(np.float32) + np.float32(0.5)) / np.float32(255)).astype(np.float32)
    assert np.array_equal((f * np.float32(255)).astype(np.int32).astype(np.uint8), q)
    return f


class Pool:
    def __init__(self, seed):
        rs = np.random.RandomState(seed)
        self.q = rs.randint(0, 256, (POOL, 84, 84)).astype(np.uint8)
        self.f_dev = torch.from_numpy(frames_for(self.q)).to(DEV)


def records(k, rs, pattern, with_final=False):
    a = rs.randint(0, 18, k).astype(np.int64)
    r = rs.choice(np.array([-1, 0, 1, 0.5, 2.25, 1e-3]), k)
    term = {"none": np.zeros(k, bool), "all": np.ones(k, bool), "random": rs.uniform(size=k) < 0.2,
            "last": np.arange(k) == k - 1}[pattern]
    fin = np.zeros(k, bool)
    if with_final:
        for j in range(1, k):
            if not term[j - 1] and not fin[j - 1] and rs.uniform() < 0.2:
                fin[j], term[j], a[j], r[j] = True, False, 0, 0.0
    return a, r, term, fin, rs.randint(0, POOL, k)


def append_all(mem, pool, a, r, term, fin, idx):
    """The records through append() one by one; a final record j and its predecessor through append_truncated."""
    k, j = len(a), 0
    state = torch.zeros(4, 84, 84, device=DEV)
    while j < k:
        state = state.clone()
        state[-1] = pool.f_dev[idx[j]]
        if j + 1 < k and fin[j + 1]:
            final_state = state.clone()
            final_state[-1] = pool.f_dev[idx[j + 1]]
            mem.append_truncated(state, int(a[j]), float(r[j]), final_state)
            j += 2
        else:
            mem.append(state, int(a[j]), float(r[j]), bool(term[j]))
            j += 1


def prepare(mem, pool, head, rs, prio_seed):
    """`head` appends, then priorities written on some leaves (so that siblings are not all the running max)."""
    a, r, term, fin, idx = records(head, rs, "random")
    append_all(mem, pool, a, r, term, fin, idx)
    mem.flush_appends()
    prs = np.random.RandomState(prio_seed)
    leaves = prs.choice(mem.capacity, min(mem.capacity, 12), replace=False) + mem.transitions.tree_start
    mem.update_priorities(leaves, prs.uniform(0.1, 4.0, leaves.size).astype(np.float32))


def as_source(q, source):
    if source == "pageable":
        return q
    t = torch.from_numpy(q)
    return t.pin_memory() if source == "pinned" else t.to(DEV)


def assert_replays_equal(got, want):
    got.flush_appends()
    want.flush_appends()
    torch.cuda.synchronize()
    g, w = got.transitions, want.transitions
    for name in ("tree", "frames", "timestep", "action", "reward", "nonterminal", "running_max"):
        assert_bits_equal(cpu(getattr(g, name)), cpu(getattr(w, name)), name)
    assert list(cpu(g.ring_state)[:4]) == list(cpu(w.ring_state)[:4]), "ring_state"
    assert (g.index, g.full, got.t) == (w.index, w.full, want.t), "host mirrors"


def run_case(cap, k, head, pattern, source, defer=False, with_final=False, queued=0, chunk_records=None, seed=0):
    from rainbow_b200.memory import ReplayMemory
    args = make_args(bootstrap_truncation=with_final)
    pool = Pool(seed)
    want = ReplayMemory(args, cap, defer_appends=defer)
    got = ReplayMemory(args, cap, defer_appends=bool(queued))
    for mem in (want, got):
        prepare(mem, pool, head, np.random.RandomState(seed + 1), seed + 2)
    rs = np.random.RandomState(seed + 3)
    if queued:   # appends left in got's defer queue: extend writes them first
        a, r, term, fin, idx = records(queued, rs, "random")
        for mem in (want, got):
            append_all(mem, pool, a, r, term, fin, idx)
        assert len(got._queue) == queued
    if chunk_records:
        got.EXTEND_CHUNK_BYTES = chunk_records * FRAME
    a, r, term, fin, idx = records(k, rs, pattern, with_final)
    append_all(want, pool, a, r, term, fin, idx)
    q = pool.q[idx]
    got.extend(as_source(q, source), a, r, term, final=fin if with_final else None)
    assert not got._queue
    assert_replays_equal(got, want)


CAPS = (14, 64, 1000)
PATTERNS = ("none", "all", "random", "last")
SOURCES = ("pageable", "pinned", "cuda")


def _ks(cap):
    return sorted({1, 7, 8, 9, cap - 1, cap, cap + 5, 3 * cap + 2})


@pytest.mark.parametrize("cap,k", [(c, k) for c in CAPS for k in _ks(c)])
def test_extend_equals_appends(cap, k):
    for h, head in enumerate((0, cap // 2 + 1, cap - 1)):
        i = _ks(cap).index(k) + h
        run_case(cap, k, head, PATTERNS[i % 4], SOURCES[(i + cap) % 3], defer=bool(i % 2), seed=cap + k + h)


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("source", SOURCES)
def test_final_records(cap, source):
    for h, head in enumerate((0, cap // 2, cap - 1)):
        for k in (2, 9, cap + 5):
            run_case(cap, k, head, "random", source, defer=bool(h % 2), with_final=True, seed=3 * cap + k + h)


@pytest.mark.parametrize("source", ("pageable", "pinned"))
@pytest.mark.parametrize("k", [40, 131])
def test_small_staging_chunks(source, k):
    """Chunks of 7 records from head 57 of 64, so the first chunk ends exactly at the wrap, then chunks of 5 with final
    records, whose pairs can straddle a chunk boundary."""
    run_case(64, k, 57, "random", source, chunk_records=7, seed=k)
    run_case(64, k, 5, "random", source, chunk_records=5, with_final=True, seed=k + 1)


@pytest.mark.parametrize("source", SOURCES)
def test_queued_appends_are_written_first(source):
    for queued in (1, 5):
        run_case(64, 30, 20, "random", source, queued=queued, seed=queued)
        run_case(14, 40, 13, "random", source, queued=queued, with_final=True, seed=queued + 9)


def test_refused_extend_writes_nothing():
    from rainbow_b200.memory import ReplayMemory
    mem = ReplayMemory(make_args(), 64, defer_appends=True)
    pool = Pool(1)
    prepare(mem, pool, 10, np.random.RandomState(0), 1)
    append_all(mem, pool, [1, 2], [0.0, 1.0], [False, False], [False, False], [0, 1])
    before = {n: cpu(getattr(mem.transitions, n)).copy() for n in ("tree", "frames", "timestep", "ring_state")}
    with pytest.raises(ValueError):
        mem.extend(torch.zeros(3, 84, 84, device=DEV), [0, 1, 2], [0.0] * 3, [False] * 3)
    with pytest.raises(ValueError):
        mem.extend(pool.q[:3], [0, 1], [0.0] * 3, [False] * 3)
    assert len(mem._queue) == 2 and mem.transitions.index == 12
    torch.cuda.synchronize()
    for n, v in before.items():
        assert_bits_equal(cpu(getattr(mem.transitions, n)), v, n)


# ---- full size ------------------------------------------------------------------------------------------------------------------
def test_full_size_fill_equals_the_reference_and_load_arrays():
    """A 1M ring filled by one extend of 1M + 3 host uint8 records: the tree equals tests/extend_ref.py bitwise, the
    records equal the inputs, and the same seed samples the same batch, bitwise, from the same data put in by load_arrays."""
    from rainbow_b200.memory import ReplayMemory
    cap, k = 1_000_000, 1_000_003
    rs = np.random.RandomState(4)
    pool = rs.randint(0, 256, (256, FRAME)).astype(np.uint8)
    idx = rs.randint(0, 256, k)
    q = pool[idx]   # 7.06 GB of host frames
    a = rs.randint(0, 18, k)
    r = rs.choice(np.array([-1.0, 0.0, 1.0]), k)
    term = rs.uniform(size=k) < 0.003
    mem = ReplayMemory(make_args(), cap, seed=21)
    mem.extend(q, a, r, term)
    del q
    ring = dict(size=cap, tree=np.zeros(mem.transitions.tree.numel(), np.float32), timestep=np.zeros(cap, np.int32),
                action=np.zeros(cap, np.int32), reward=np.zeros(cap, np.float32), nonterminal=np.zeros(cap, np.uint8),
                index=0, full=False, t=0, max=np.float32(1.0))
    want = extend_ref.extend(ring, a, r.astype(np.float32), term.astype(np.uint8))
    torch.cuda.synchronize()
    tr = mem.transitions
    assert_bits_equal(cpu(tr.tree), want["tree"], "tree")
    for key in ("timestep", "action", "reward", "nonterminal"):
        assert_bits_equal(cpu(getattr(tr, key)), want[key], key)
    assert (tr.index, tr.full, mem.t) == (want["index"], want["full"], want["t"])
    assert list(cpu(tr.ring_state)[:4]) == [want["index"], 1, want["t"], k]
    slots = np.arange(cap)
    j = np.where(slots < k - cap, slots + cap, slots)   # the record each slot holds
    pool_dev, src = torch.from_numpy(pool).to(DEV), torch.from_numpy(idx[j]).to(DEV)
    for s0 in range(0, cap, 100_000):
        assert torch.equal(tr.frames[s0:s0 + 100_000], pool_dev[src[s0:s0 + 100_000]]), f"frames from slot {s0}"

    other = ReplayMemory(make_args(), cap, seed=21)
    other.transitions.load_arrays(sum_tree=want["tree"], timestep=want["timestep"], action=want["action"],
                                  reward=want["reward"], nonterminal=want["nonterminal"], index=want["index"], full=True,
                                  t_episode=want["t"], max_value=1.0)
    other.transitions.frames.copy_(tr.frames)
    other.t = want["t"]
    for _ in range(3):
        x, y = mem.sample(32), other.sample(32)
        for u, v in zip(x, y):
            assert_bits_equal(cpu(u), cpu(v), "sample")


# ---- offline end to end ---------------------------------------------------------------------------------------------------------
def test_offline_cql_from_arrays_graph_equals_eager():
    """A replay filled by extend from a seeded dataset (uniform sampling, priority_exponent = 0), then CQL updates with no
    acting: graph replay equals eager update by update, and both equal a replay filled by append."""
    from rainbow_b200.agent import Agent
    from rainbow_b200.memory import ReplayMemory
    A, cap, k = 6, 2048, 2500
    rs = np.random.RandomState(11)
    acts = rs.randint(0, A, k)
    q = (rs.uniform(0.0, 0.2, (k, 84, 84)) * 255).astype(np.uint8)
    for j in range(k):
        q[j, acts[j] * 14:(acts[j] + 1) * 14, :] += 200
    r = rs.randint(-1, 2, k).astype(np.float64)
    term = rs.uniform(size=k) < 0.02
    agents, mems = [], []
    for graph in (True, False):
        args = make_args(priority_exponent=0.0, batch_size=32, architecture="data-efficient", hidden_size=64,
                         cql_alpha=2.0, learning_rate=1e-3, cuda_graph=graph)
        mem = ReplayMemory(args, cap, seed=7)
        mem.extend(q, acts, r, term)
        torch.manual_seed(5)
        agents.append(Agent(args, FakeEnv(A)))
        mems.append(mem)
    ga, ea = agents
    for step in range(8):
        for ag, mem in zip(agents, mems):
            ag.reset_noise()
            ag.learn(mem)
        assert_bits_equal(cpu(ga.last_loss), cpu(ea.last_loss), f"loss of update {step}")
        assert_bits_equal(cpu(ga.last_cql_gap), cpu(ea.last_cql_gap), f"gap of update {step}")
    assert ga._graphs and not ea._graphs
    assert np.isfinite(cpu(ga.optimiser.flat_param)).all()
    for key in ("flat_param", "exp_avg", "exp_avg_sq"):
        assert_bits_equal(cpu(getattr(ga.optimiser, key)), cpu(getattr(ea.optimiser, key)), key)
