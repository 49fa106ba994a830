"""Exact resume: Agent.save_checkpoint / Agent.load_checkpoint (rainbow_b200/checkpoint.py) on the GPU.

* A run that saves after 5 updates, builds a fresh Agent + ReplayMemory, loads and does 7 more agrees bitwise with a run of
  12 updates that never stopped: every loss, the parameters, target net, Adam state, sum tree, ring state, sampling and
  noise streams, and all 12 statistics records.  Both runs append transitions between updates (some still queued by
  defer_appends at the save, some ending episodes) and refresh the target net once before the save.
* Loading into the same objects rolls a run back and replays the same captured graph.
* Every refusal raises and leaves all device arrays and host fields unchanged; a failed save leaves nothing behind.
* rng="numpy" sampling resumes bitwise when the caller restores numpy's global generator itself.
* Two data-parallel ranks resume bitwise each; a checkpoint corrupted on one rank, or whose rank directories come from
  different saves, makes both raise.
Like the other trajectory tests this one runs with deterministic cuDNN algorithms (DESIGN.md §9)."""
import json
import os

import numpy as np
import pytest
import torch

from test_gpu_parity import DEV, FakeEnv, cpu, make_args, synthetic_ring

pytestmark = pytest.mark.gpu

CAP = 8192
SAVE_AT, TOTAL = 5, 12


@pytest.fixture(autouse=True)
def deterministic_cudnn():
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = old


def _agent(seed=5, **kw):
    from rainbow_b200.agent import Agent
    torch.manual_seed(seed)
    kw.setdefault("learn_stats", 16)
    return Agent(make_args(**kw), FakeEnv(6))


def _memory(**kw):
    mem, _ = synthetic_ring(CAP, seed=3, args=dict(), defer_appends=True, **kw)
    mem.seed = 99
    return mem


def _fresh_memory(**kw):
    """A memory built as a resuming driver builds it: empty, another seed."""
    from rainbow_b200.memory import ReplayMemory
    return ReplayMemory(make_args(), CAP, seed=12345, defer_appends=True, **kw)


def _appends(mem, step):
    """Transitions between updates: odd steps queue theirs (defer_appends), even steps write them at once and end an
    episode.  Fewer than ReplayMemory.APPEND_BATCH per step, so a queue is still pending at the next learn() / save."""
    rs = np.random.RandomState(1000 + step)
    if step % 2 == 0:
        mem.flush_appends()
    mem.defer_appends = step % 2 == 1
    for i in range(3):
        st = torch.from_numpy(rs.uniform(0, 1, (4, 84, 84)).astype(np.float32)).to(DEV)
        mem.append(st, int(rs.randint(0, 6)), float(rs.randint(-1, 2)), step % 2 == 0 and i == 2)


def _before_update(ag, mem, step, pending):
    _appends(mem, step)
    ag.reset_noise()
    if not pending:
        ag.online_net.flush_noise()        # as an act() between reset_noise() and learn() would


def _update(ag, mem, step, losses):
    ag.learn(mem)
    losses.append(ag.last_loss.clone())
    if step == 2:
        ag.update_target_net()             # target != online at the checkpoint


def _state(ag, mem, losses):
    torch.cuda.synchronize()
    opt, tr = ag.optimiser, mem.transitions
    dev = dict(losses=torch.stack(losses), flat_param=opt.flat_param, exp_avg=opt.exp_avg, exp_avg_sq=opt.exp_avg_sq,
               step_count=opt.step_count, tree=tr.tree, running_max=tr.running_max, rng_counter=mem._rng_counter,
               ring_state=tr.ring_state[:4], frames=tr.frames, timestep=tr.timestep)
    for n, p in ag.target_net.named_parameters():
        dev["target." + n] = p
    for tag, net in (("online", ag.online_net), ("target", ag.target_net)):
        dev[tag + ".noise_counter"], dev[tag + ".f_in"], dev[tag + ".f_out"] = net._noise_counter, net._f_in, net._f_out
        dev.update((f"{tag}.{n}", b) for n, b in net.named_buffers() if n.endswith("_epsilon"))
    out = {k: cpu(v).copy() for k, v in dev.items()}
    out["host"] = (tr.index, tr.full, mem.t, ag.online_net.noise_seed, ag.target_net.noise_seed)
    return out


def _assert_same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if k == "host":
            assert a[k] == b[k], k
        else:
            assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
            assert a[k].tobytes() == b[k].tobytes(), f"{k} differs between the resumed and the uninterrupted run"


def _assert_records_same(ra, rb, n):
    assert ra["dropped"] == rb["dropped"] == 0
    assert ra["update"].tolist() == rb["update"].tolist() == list(range(n))
    for k in ra:
        if k != "dropped":
            assert np.ascontiguousarray(ra[k]).tobytes() == np.ascontiguousarray(rb[k]).tobytes(), k


CASES = {
    "fused-pending": dict(kw=dict(), pending=True),
    "fused-flushed": dict(kw=dict(), pending=False),
    "library-flushed": dict(kw=dict(fused_head=False), pending=False),
    "batch64-large-backward": dict(kw=dict(batch_size=64), pending=True),
    "data-efficient-h256": dict(kw=dict(architecture="data-efficient", hidden_size=256), pending=True),
    # graph replay != eager on this path is a known defect (DESIGN.md §4): both sides run eagerly
    "library-pending-eager": dict(kw=dict(fused_head=False, cuda_graph=False), pending=True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_resume_equals_never_stopping(case, tmp_path):
    kw, pending = CASES[case]["kw"], CASES[case]["pending"]
    ag, mem = _agent(**kw), _memory()
    if case.startswith("batch64"):
        assert ag.batch_size > 32, "past k_head_bwd1's limit of 32 rows: the large-batch layer-1 kernels"
    if case.startswith(("fused", "batch64")):
        assert ag._fused_path(ag.batch_size)
    if case.startswith("library"):
        assert not ag._fused_path(ag.batch_size)
    losses = []
    for step in range(TOTAL):
        _before_update(ag, mem, step, pending)
        _update(ag, mem, step, losses)
    if kw.get("cuda_graph", True):
        assert set(ag._graphs) == {pending}
    run_a, rec_a = _state(ag, mem, losses), ag.learn_stats()

    ag, mem = _agent(**kw), _memory()
    losses = []
    for step in range(SAVE_AT):
        _before_update(ag, mem, step, pending)
        _update(ag, mem, step, losses)
    _before_update(ag, mem, SAVE_AT, pending)
    assert mem._queue, "transitions queued at the save"
    assert ag.online_net._noise_pending == pending
    ag.save_checkpoint(str(tmp_path / "ck"), mem)
    del ag, mem
    ag, mem = _agent(seed=77, **kw), _fresh_memory()
    ag.load_checkpoint(str(tmp_path / "ck"), mem)
    for step in range(SAVE_AT, TOTAL):
        if step > SAVE_AT:
            _before_update(ag, mem, step, pending)
        _update(ag, mem, step, losses)
    _assert_same(run_a, _state(ag, mem, losses))
    _assert_records_same(rec_a, ag.learn_stats(), TOTAL)


def test_rollback_in_place_replays_the_same_graph(tmp_path):
    ag, mem = _agent(), _memory()
    losses = []
    for step in range(4):                  # warm-up x2, capture, replay
        _before_update(ag, mem, step, True)
        _update(ag, mem, step, losses)
    _before_update(ag, mem, 4, True)
    assert ag.learn_stats()["update"].tolist() == [0, 1, 2, 3]
    ag.save_checkpoint(str(tmp_path / "ck"), mem)
    graph = ag._graphs[True][0]

    def run():
        out = []
        for step in range(4, 7):
            if step > 4:
                _before_update(ag, mem, step, True)
            _update(ag, mem, step, out)
        return _state(ag, mem, out), ag.learn_stats()

    first, rec1 = run()
    ag.load_checkpoint(str(tmp_path / "ck"), mem)
    assert ag._graphs[True][0] is graph
    second, rec2 = run()
    assert set(ag._graphs) == {True} and ag._graphs[True][0] is graph, "no recapture"
    _assert_same(first, second)
    assert rec1["update"].tolist() == rec2["update"].tolist() == [4, 5, 6]
    for k in rec1:
        assert np.ascontiguousarray(rec1[k]).tobytes() == np.ascontiguousarray(rec2[k]).tobytes(), k


# ---- refusals -------------------------------------------------------------------------------------------------------------
def _small(**kw):
    d = dict(architecture="data-efficient", hidden_size=64, batch_size=8, learn_stats=4)
    d.update(kw)
    return d


def _small_pair(cap=1024, **kw):
    from rainbow_b200.memory import ReplayMemory
    ag = _agent(**_small(**kw))
    mem = ReplayMemory(make_args(**{k: v for k, v in kw.items() if k == "history_length"}), cap, seed=4)
    return ag, mem


def _filled_small(tmp_path):
    ag, mem = _small_pair()
    tr = mem.transitions
    tr.load_arrays(timestep=np.arange(1024) % 50, action=np.arange(1024) % 6, reward=np.ones(1024),
                   nonterminal=np.ones(1024), index=10, full=True, t_episode=11)
    tr.frames.fill_(7)
    tr.update(np.arange(1024) + tr.tree_start, np.full(1024, 0.5, np.float32))
    for _ in range(3):
        ag.reset_noise()
        ag.learn(mem)
    ag.save_checkpoint(str(tmp_path / "ck"), mem)
    for _ in range(2):                     # the live state moves on: a refused load must not bring back the saved one
        ag.reset_noise()
        ag.learn(mem)
    return ag, mem


def _snapshot(ag, mem):
    from rainbow_b200 import checkpoint as ck
    torch.cuda.synchronize()
    arrays = dict(ck._learner_arrays(ag), **(ck._replay_arrays(mem) if mem is not None else {}))
    snap = {k: cpu(v).tobytes() for k, v in arrays.items()}
    snap["flat_grad"] = cpu(ag.optimiser.flat_grad).tobytes()
    host = (ag._learn_calls, ag.online_net.noise_seed, ag.target_net.noise_seed, ag.online_net._noise_pending,
            ag.learn_stats_capacity, ag._stats["read"] if ag._stats else None)
    if mem is not None:
        host += (mem.transitions.index, mem.transitions.full, mem.t, mem.seed, mem.priority_weight, len(mem._queue))
    return snap, host


def _refused(ag, mem, path, match=None):
    from rainbow_b200 import RainbowB200Error
    before = _snapshot(ag, mem)
    with pytest.raises(RainbowB200Error, match=match):
        ag.load_checkpoint(path, mem)
    after = _snapshot(ag, mem)
    assert before[1] == after[1], "host fields changed by a refused load"
    changed = [k for k in before[0] if before[0][k] != after[0][k]]
    assert not changed, f"device arrays changed by a refused load: {changed}"


@pytest.mark.parametrize("what", ["hidden_size", "atoms", "actions", "history_length", "capacity"])
def test_structure_mismatch_is_refused(what, tmp_path):
    from rainbow_b200.agent import Agent
    from rainbow_b200.memory import ReplayMemory
    _filled_small(tmp_path)
    kw = dict(hidden_size=dict(hidden_size=128), atoms=dict(atoms=41), history_length=dict(history_length=3)).get(what, {})
    cap = 2048 if what == "capacity" else 1024
    torch.manual_seed(3)
    ag = Agent(make_args(**_small(**kw)), FakeEnv(4 if what == "actions" else 6))
    mem = ReplayMemory(make_args(**{k: v for k, v in kw.items() if k == "history_length"}), cap, seed=4)
    _refused(ag, mem, str(tmp_path / "ck"), match={"actions": "actions", "capacity": "replay"}.get(what, what))


def _reseal(man_path, man):
    """Write an edited manifest with a matching digest, as a writer of those values would."""
    from rainbow_b200 import checkpoint as ck
    man["digest"] = ck._digest(man)
    json.dump(man, open(man_path, "w"))


def _corrupt(directory, what):
    man_path = os.path.join(directory, "manifest.json")
    man = json.load(open(man_path))
    if what == "version":
        man["version"] += 1
        _reseal(man_path, man)
    elif what == "world":
        man["world_size"], man["rank"] = 2, 0          # rank 0's directory of a two-rank run
        _reseal(man_path, man)
    elif what == "missing":
        os.remove(os.path.join(directory, "optimiser.exp_avg_sq.npy"))
    elif what == "manifest-edit":                      # a hand edit without a matching digest
        man["replay"]["index"] = 3
        json.dump(man, open(man_path, "w"))
    elif what == "index-range":
        man["replay"]["index"] = man["structure"]["replay"]["capacity"]
        _reseal(man_path, man)
    elif what == "scalar-missing":
        del man["learner"]["optimiser_step"]
        _reseal(man_path, man)
    elif what == "scalar-type":
        man["learner"]["online_noise_pending"] = "yes"
        _reseal(man_path, man)
    elif what == "file-name":
        man["arrays"]["online.flat_param"]["file"] = "../rank0/online.flat_param.npy"
        _reseal(man_path, man)
    else:
        path = os.path.join(directory, "replay.frames.npy" if what == "flip" else "online.flat_param.npy")
        raw = bytearray(open(path, "rb").read())
        if what == "flip":
            raw[len(raw) // 2] ^= 0x01
        else:
            raw = raw[:len(raw) - 100]
        open(path, "wb").write(bytes(raw))


REFUSALS = dict(version="version", flip="SHA-256", truncated="truncated", missing="missing", world="rank",
                **{"manifest-edit": "digest", "index-range": "replay.index", "scalar-missing": "optimiser_step",
                   "scalar-type": "online_noise_pending", "file-name": "naming rule"})


@pytest.mark.parametrize("what", list(REFUSALS))
def test_corrupt_checkpoint_is_refused(what, tmp_path):
    ag, mem = _filled_small(tmp_path)
    _corrupt(str(tmp_path / "ck" / "rank0"), what)
    _refused(ag, mem, str(tmp_path / "ck"), match=REFUSALS[what])


def test_replay_required_and_learner_only(tmp_path):
    ag, mem = _filled_small(tmp_path)
    ag.save_checkpoint(str(tmp_path / "learner"))            # no replay in it
    _refused(ag, mem, str(tmp_path / "learner"), match="no replay")
    ag.load_checkpoint(str(tmp_path / "ck"))                  # a checkpoint with a replay also restores the learner alone


def test_failed_save_leaves_nothing_and_the_previous_checkpoint_loads(tmp_path, monkeypatch):
    from rainbow_b200 import checkpoint as ck
    ag, mem = _filled_small(tmp_path)
    real, calls = ck.write_array, []

    def failing(path, src, staging):
        if calls:
            raise OSError("preempted")
        calls.append(path)
        return real(path, src, staging)

    monkeypatch.setattr(ck, "write_array", failing)
    with pytest.raises(OSError):
        ag.save_checkpoint(str(tmp_path / "next"), mem)
    assert calls and not os.path.exists(tmp_path / "next")
    with pytest.raises(OSError):
        calls.clear()
        ag.save_checkpoint(str(tmp_path / "ck"), mem)       # over the previous one: it stays whole
    monkeypatch.setattr(ck, "write_array", real)
    assert sorted(os.listdir(tmp_path / "ck")) == ["rank0"]
    ag.load_checkpoint(str(tmp_path / "ck"), mem)


def test_pickle_layout_unchanged():
    """ReplayMemory.__getstate__ now reads the persistent-field list the checkpoint shares: same keys, order and values."""
    import pickle
    mem = _memory()
    tr = mem.transitions
    old = dict(
        version=1, capacity=mem.capacity, history=mem.history, discount=mem.discount, n=mem.n,
        priority_weight=mem.priority_weight, priority_exponent=mem.priority_exponent, t=mem.t, rng=mem.rng,
        seed=mem.seed, max_attempts=mem.max_attempts, strict=mem.strict, device=str(mem.device),
        rng_counter=int(mem._rng_counter.item()), index=tr.index, full=tr.full, max=tr.max,
        sum_tree=tr.sum_tree, frames=tr.frames.cpu().numpy(), timestep=tr.timestep.cpu().numpy(),
        action=tr.action.cpu().numpy(), reward=tr.reward.cpu().numpy(), nonterminal=tr.nonterminal.cpu().numpy())
    assert pickle.dumps(mem.__getstate__()) == pickle.dumps(old)


# ---- host generators are the caller's -------------------------------------------------------------------------------------
def test_numpy_rng_memory_resumes_with_the_callers_generator(tmp_path):
    def fresh_mem():
        m, _ = synthetic_ring(CAP, seed=3, args=dict(), rng="numpy")
        return m

    kw = dict(architecture="data-efficient", hidden_size=256)
    np.random.seed(11)
    ag, mem = _agent(**kw), fresh_mem()
    losses = []
    for step in range(8):
        ag.reset_noise()
        _update(ag, mem, step, losses)
    run_a = _state(ag, mem, losses)

    np.random.seed(11)
    ag, mem = _agent(**kw), fresh_mem()
    losses = []
    for step in range(3):
        ag.reset_noise()
        _update(ag, mem, step, losses)
    ag.save_checkpoint(str(tmp_path / "ck"), mem)
    np_state = np.random.get_state()        # the caller saves its own generators
    np.random.seed(0)
    ag, mem = _agent(seed=77, **kw), fresh_mem()
    ag.load_checkpoint(str(tmp_path / "ck"), mem)
    np.random.set_state(np_state)
    for step in range(3, 8):
        ag.reset_noise()
        _update(ag, mem, step, losses)
    _assert_same(run_a, _state(ag, mem, losses))


# ---- two data-parallel ranks ----------------------------------------------------------------------------------------------
_DP_WORKER = r"""
import os, sys, json, shutil
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
out_dir = sys.argv[2]
from rainbow_b200.dist import init_from_env
ngpu = torch.cuda.device_count()
backend = "nccl" if ngpu >= 2 else "gloo"          # one GPU: both ranks share it, gloo moves the CUDA tensors
if backend == "gloo":
    os.environ["LOCAL_RANK"] = "0"
rank, world, local = init_from_env(backend)
torch.backends.cudnn.deterministic = True
from test_gpu_parity import FakeEnv, make_args, synthetic_ring
from rainbow_b200 import RainbowB200Error
from rainbow_b200.agent import Agent
from rainbow_b200.memory import ReplayMemory
dev = torch.device("cuda", local)
torch.cuda.set_device(dev)

def same_everywhere(x, what):
    a = torch.as_tensor(np.asarray(x, np.float64)).to(dev)
    lo, hi = a.clone(), a.clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN); dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    assert torch.equal(lo, hi), what

def build(peer, seed=7):
    torch.manual_seed(seed)
    args = make_args(device=dev, cuda_graph=backend == "nccl", architecture="data-efficient", hidden_size=64, batch_size=8,
                     learn_stats=8, peer_optimizer=peer)
    return Agent(args, FakeEnv(4))

def state(ag, mem, losses):
    torch.cuda.synchronize()
    opt = ag.optimiser
    ts = [torch.stack(losses), opt.flat_param, opt.exp_avg, opt.exp_avg_sq, opt.step_count, mem.transitions.tree,
          mem._rng_counter] + [p for p in ag.target_net.parameters()]
    return [t.detach().cpu().numpy().tobytes() for t in ts]

variants = [False] + ([True] if ngpu >= 2 else [])   # the peer-memory optimiser needs a GPU per rank
for peer in variants:
    ck = os.path.join(out_dir, f"peer{int(peer)}")
    ag, losses = build(peer), []
    mem, _ = synthetic_ring(1024, seed=10, device=str(dev), args=dict(device=dev))
    for k in range(8):
        ag.reset_noise(); ag.learn(mem); losses.append(ag.last_loss.clone())
    run_a = state(ag, mem, losses)
    same_everywhere(ag.optimiser.flat_param.cpu().numpy(), "parameters identical across ranks")

    ag, losses = build(peer), []
    mem, _ = synthetic_ring(1024, seed=10, device=str(dev), args=dict(device=dev))
    for k in range(3):
        ag.reset_noise(); ag.learn(mem); losses.append(ag.last_loss.clone())
    ag.reset_noise()
    ag.save_checkpoint(ck, mem)
    dist.barrier()
    assert sorted(os.listdir(ck)) == ["rank0", "rank1"]
    ag = build(peer, seed=99)
    mem = ReplayMemory(make_args(device=dev), 1024, seed=5)
    ag.load_checkpoint(ck, mem)
    for k in range(3, 8):
        if k > 3:
            ag.reset_noise()
        ag.learn(mem); losses.append(ag.last_loss.clone())
    run_b = state(ag, mem, losses)
    bad = [i for i, (a, b) in enumerate(zip(run_a, run_b)) if a != b]
    assert not bad, f"rank {rank}: resumed run differs in {bad}"
    same_everywhere(ag.optimiser.flat_param.cpu().numpy(), "parameters identical across ranks after the resume")

    # a later save whose rank-1 directory is swapped for the earlier save's (as a preemption between the ranks' renames
    # would leave it): each directory is complete, but every rank must refuse to restore a different update
    later = ck + "-later"
    ag.reset_noise(); ag.learn(mem)
    ag.save_checkpoint(later, mem)
    dist.barrier()
    if rank == 1:
        shutil.rmtree(os.path.join(later, "rank1")); shutil.copytree(os.path.join(ck, "rank1"), os.path.join(later, "rank1"))
    dist.barrier()
    before, calls = ag.optimiser.flat_param.clone(), ag._learn_calls
    try:
        ag.load_checkpoint(later, mem)
        raise AssertionError("rank directories of different saves were accepted")
    except RainbowB200Error as e:
        assert "different saves" in str(e), str(e)
    assert torch.equal(before, ag.optimiser.flat_param) and ag._learn_calls == calls
    print(f"rank{rank}mixed-refused peer={peer}", flush=True)

    dist.barrier()
    if rank == 1:                                       # one rank's copy is corrupt: every rank must refuse
        man = json.load(open(os.path.join(ck, "rank1", "manifest.json")))
        path = os.path.join(ck, "rank1", man["arrays"]["online.flat_param"]["file"])
        raw = bytearray(open(path, "rb").read()); raw[-5] ^= 0x40; open(path, "wb").write(bytes(raw))
    dist.barrier()
    before = ag.optimiser.flat_param.clone()
    try:
        ag.load_checkpoint(ck, mem)
        raise AssertionError("a corrupt checkpoint on one rank was accepted")
    except RainbowB200Error as e:
        assert ("another rank" in str(e)) == (rank == 0), str(e)
    assert torch.equal(before, ag.optimiser.flat_param)
    print(f"rank{rank}ok peer={peer}", flush=True)
dist.barrier()
dist.destroy_process_group()
print(f"rank{rank}done backend={backend}", flush=True)
"""


def test_two_rank_resume(tmp_path):
    """Data parallel (torchrun world 2; NCCL + graphs with two GPUs, else both ranks on this GPU with gloo, eagerly): each
    rank resumes bitwise against its own uninterrupted run, parameters stay identical across ranks, and a checkpoint
    corrupted on one rank makes every rank raise.  With a GPU per rank also on the peer-memory optimiser (sharded moments)."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "dp_checkpoint_worker.py"
    script.write_text(_DP_WORKER)
    (tmp_path / "ck").mkdir()
    port = 29650 + os.getpid() % 150
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(script), root, str(tmp_path / "ck")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, OMP_NUM_THREADS="1"))
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-4000:]
    assert out.stdout.count("done backend=") == 2 and out.stdout.count("ok peer=False") == 2, out.stdout
    assert out.stdout.count("mixed-refused peer=False") == 2, out.stdout
