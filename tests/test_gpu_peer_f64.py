"""The peer-memory optimiser (csrc/rb_peer.cu: rb_peer_reduce, rb_peer_adam_gather, rb_peer_clip_adam) against the
stage-by-stage reference of tests/peer_ref.py, with W = 1, 2, 4 and 8 ranks emulated on one GPU (peer_ref.World: the host
plays the part of the ranks that have not launched yet, and asserts before every launch that nothing it waits on is
missing).

Layouts, each at every W (the per-rank part of a segment is the same at every W, so the loop edges are too):
 * one segment through rb_peer_clip_adam, two segments through rb_peer_reduce (segment 0 on a side stream, as in the
   learner) + rb_peer_adam_gather, segment 0 after segment 1 in the flat buffer (it does not start at 0);
 * parts of one quad (P = 4W); of exactly 64 * 256 * 4 quads, one full unrolled round of the reduce's 64 CTAs (UN = 4
   grid strides), and of one quad more; of more than 592 * 256 quads, so k_peer_adam's grid-stride loop takes a second
   round; of quad counts that are not a multiple of 256;
 * the learner's own layouts (canonical / 512: P = 6 868 928; data-efficient / 256), built as FusedClipAdam builds them.
Five steps each (t = 1 ... 5: epochs and the self-resetting tickets advance): gradients clipped, unclipped, all zero
(coef 1), clipped, unclipped.  After every step peer_ref.check_step asserts gred bitwise, every segment's squared norm
within 1e-12, every norm slot and the norm bitwise on every rank, parameters and moments within adam_ref.TAU, the
parameters bitwise the same on every rank, step_count and epoch, the guards, every flag block and the tickets.

Also: a graph capture of rb_peer_adam_gather replays bitwise like the eager call, and, on a host with 2+ GPUs,
PeerOptimizerState over real symmetric memory (torchrun) passes the same checks."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import peer_ref as PR
from test_gpu_parity import DEV

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROUND = 64 * 256 * 4          # quads: one full round of the reduce (64 CTAs x 256 threads x UN = 4 strides)
ADAM_ROUND = 592 * 256        # quads: one grid stride of k_peer_adam at its CTA cap

# name -> per-rank part of each segment in floats (segment 0 first; one entry: one segment), or a learner architecture
LAYOUTS = {
    "one-quad": (4,),
    "one-quad-2seg": (4, 4),
    "round": (4 * ROUND,),
    "round+1-2seg": (4 * (ROUND + 1), 4 * ROUND),
    "adam-2nd-round": (4 * (ADAM_ROUND + 37),),
    "odd-quads-2seg": (4 * (3 * 256 + 5), 4 * (ADAM_ROUND + 1)),
    "canonical-512": "canonical",
    "data-efficient-256": "data-efficient",
}


def lib():
    from rainbow_b200 import _lib
    return _lib.load()


def segments_of(layout, world):
    spec = LAYOUTS[layout]
    if isinstance(spec, str):
        segs = PR.learner_segments(spec)
        if spec == "canonical":
            assert segs[0][1] == 6_868_928
        return segs
    if len(spec) == 1:
        return [(0, world * spec[0])]
    head, body = world * spec[0], world * spec[1]
    return [(body, body + head), (0, body)]


def new_world(layout, world, seed):
    w = PR.World(world, segments_of(layout, world), DEV, lib())
    p0 = torch.from_numpy(np.random.default_rng(seed).standard_normal(w.P, dtype=np.float32) * np.float32(0.05))
    for rk in w.ranks:
        rk["param"][:w.P].copy_(p0)
    torch.cuda.synchronize()
    return w


def load_grads(w, seed, t, kind):
    grads = [PR.step_grad(seed, t, q, w.P, kind) for q in range(w.W)]
    for rk, g in zip(w.ranks, grads):
        rk["grad"][:w.P].copy_(torch.from_numpy(g))
    torch.cuda.synchronize()
    return grads


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_peer_optimiser_f64(layout, world):
    seed = 100 * list(LAYOUTS).index(layout) + world
    w = new_world(layout, world, seed)
    side = torch.cuda.Stream(device=DEV)
    before = w.snapshot()
    for t, kind in enumerate(PR.STEP_KINDS, 1):
        grads = load_grads(w, seed, t, kind)
        w.step(PR.HYPER, side)
        after = w.snapshot()
        coef = PR.check_step(after, before, grads, w.segments, t, PR.HYPER, DEV)
        assert (coef < 1.0) == (kind == "clip"), f"step {t} ({kind}): reference clip coefficient {coef}"
        before = after


def test_peer_adam_gather_graph_replay_equals_eager():
    """Rank 0's rb_peer_adam_gather of the second step, captured in a graph and replayed, leaves every rank's state
    bitwise as the eager call does, under the same emulated flags and norm slots."""
    w = new_world("odd-quads-2seg", 2, 7)
    side, cur = torch.cuda.Stream(device=DEV), torch.cuda.current_stream()
    load_grads(w, 7, 1, "clip")
    w.step(PR.HYPER, side)
    load_grads(w, 7, 2, "noclip")
    w.reduce_all(side)
    state, launched = w.state(), {k: set(v) for k, v in w.launched.items()}
    runs = []
    for graphed in (False, True):
        w.restore(state)
        w.launched = {k: set(v) for k, v in launched.items()}
        w.prepare_adam(0)
        if graphed:
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                w.launch_adam(0, PR.HYPER, torch.cuda.current_stream())
            graph.replay()
        else:
            w.launch_adam(0, PR.HYPER, cur)
        torch.cuda.synchronize()
        assert int(w.ranks[0]["step_count"].item()) == 2 and int(w.ranks[0]["epoch"].item()) == 2
        runs.append(w.state())
    moved = 0
    for r, (eager, replayed) in enumerate(zip(*runs)):
        for k in eager:
            assert torch.equal(eager[k].view(torch.uint8), replayed[k].view(torch.uint8)), f"rank {r} {k}: replay != eager"
        moved += not torch.equal(eager["param"].view(torch.uint8), state[r]["param"].view(torch.uint8))
    assert moved == 2, "rank 0's parts reach both ranks' parameters"


# One process per GPU over real symmetric memory: every rank all-gathers every rank's gradients and state after each step
# and runs peer_ref.check_step on them.
_REAL_WORKER = r"""
import os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
from rainbow_b200.dist import init_from_env
from rainbow_b200.peer import PeerOptimizerState
import peer_ref as PR
rank, world, local = init_from_env("nccl")
dev = torch.device("cuda", local)
torch.cuda.set_device(dev)
segments = PR.learner_segments("canonical")
P = segments[0][1]
peer = PeerOptimizerState(P, dev, segments=segments)
peer.flat_param.copy_(torch.from_numpy(np.random.default_rng(5).standard_normal(P, dtype=np.float32) * np.float32(0.05)))
side, cur = torch.cuda.Stream(device=dev), torch.cuda.current_stream()
W = world
flags = peer.buf[peer._off[2]:peer._off[2] + 32 * W].view(torch.int64)
norms = peer.buf[peer._off[3]:peer._off[3] + 8 * W].view(torch.float64)
seg_norm = peer._scratch.view(torch.float64)[PR.SEG_NORM_AT:PR.SEG_NORM_AT + 2]
tickets = peer._scratch.view(torch.int32)[PR.TICKETS_AT:PR.TICKETS_AT + PR.N_TICKETS]


def gather(t):
    out = [torch.empty_like(t) for _ in range(W)]
    dist.all_gather(out, t.contiguous())
    return [o.cpu().numpy() for o in out]


def snapshot():
    torch.cuda.synchronize()
    f = dict(param=peer.flat_param, gred=peer.gred, exp_avg=peer.exp_avg, exp_avg_sq=peer.exp_avg_sq, step_count=peer.step_count,
             epoch=peer.epoch, grad_norm=peer.grad_norm, norms=norms, flags=flags, seg_norm=seg_norm, tickets=tickets)
    g = {k: gather(v) for k, v in f.items()}
    snaps = [{k: g[k][r] for k in g} for r in range(W)]
    for s in snaps:
        s["step_count"], s["epoch"] = int(s["step_count"][0]), int(s["epoch"][0])
    return snaps


before = snapshot()
for t, kind in enumerate(PR.STEP_KINDS[:3], 1):
    peer.flat_grad.copy_(torch.from_numpy(PR.step_grad(11, t, rank, P, kind)))
    side.wait_stream(cur)
    with torch.cuda.stream(side):
        peer.reduce_segment(0)
    cur.wait_stream(side)
    max_norm, lr, betas, eps = PR.HYPER
    peer.step(max_norm, lr, betas, eps)
    torch.cuda.synchronize()
    grads = gather(peer.flat_grad)
    after = snapshot()
    coef = PR.check_step(after, before, grads, segments, t, PR.HYPER, dev)
    assert (coef < 1.0) == (kind == "clip"), (t, kind, coef)
    before = after
dist.barrier()
print(f"rank {rank}: peer optimiser over {W} GPUs matches peer_ref", flush=True)
dist.destroy_process_group()
"""


def test_peer_optimiser_real_ranks(tmp_path):
    """PeerOptimizerState on the learner's canonical layout over real symmetric memory, one rank per GPU (2, 4 or 8),
    three steps, every rank checked against peer_ref."""
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip(f"real peer memory needs 2+ GPUs; this host has {n}")
    nproc = max(k for k in (2, 4, 8) if k <= n)
    script = tmp_path / "peer_worker.py"
    script.write_text(_REAL_WORKER)
    port = 29850 + os.getpid() % 100
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr",
           "127.0.0.1", "--master-port", str(port), str(script), ROOT]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, OMP_NUM_THREADS="1"))
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-4000:]
    assert out.stdout.count("matches peer_ref") == nproc, out.stdout[-2000:]
