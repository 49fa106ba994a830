"""An emulated world of W ranks on one GPU for the peer-memory optimiser (csrc/rb_peer.cu), and its reference, stage by
stage.

The kernels see the other ranks only through arrays of W device pointers (every rank's gradients, parameters, flag
block and norm block), and they wait for the other ranks only through `flag >= epoch` loads from device memory
(`wait_flags`).  So W ranks can be W sets of allocations on one device, launched one after another on one stream, with
the host playing the part of every rank that has not launched yet in the current phase: before a launch of rank r it
writes what those ranks would have published (their flags and, for the norm exchange, their partial squared norm read
from their own scratch).  What the ranks that have already launched published is left to their kernels.  Then it reads
rank r's flag block back and asserts that every flag the launch will wait on, other than the ones the launch writes
itself, is already set.  A mistake in the emulation, or a kernel that fails to publish a flag, is an assertion on the
host, never a kernel spinning on a flag.

Reference, each stage from the kernel's own output of the stage before:
  gred       bitwise fl32(((0 + g_0) + g_1) + ... + g_{W-1}) * fl32(1/W) on the owned part (numpy float32 in rank order;
             the kernel starts its sum from +0.0 too, which matters only for -0.0);
  seg_norm   the float64 sum of squares of the kernel's gred part, within SEG_NORM_RTOL (derived below);
  norms      every slot norms[r][q] holds, bitwise, rank q's partial 0.0 + seg_norm[0] (+ seg_norm[1]) from its scratch;
  grad_norm  bitwise fl32(sqrt(norms[r][0] + ... + norms[r][W-1])) summed in q order from 0.0, the same bits on every rank;
  p, m, v    tests/adam_ref.py's clip_adam(p, gred, m, v, t - 1, 1.0, ...) within adam_ref.TAU, the moments through
             the shard mapping of PeerOptimizerState.shard_slices.

SEG_NORM_RTOL.  The square of an fp32 value is exact in double (two 24-bit significands), so only the additions round.
k_peer_reduce runs c = min(ceil(q / 256), 64) CTAs of 256 threads over a part of q quads.  A thread adds the 4 squares
of each of its at most k = ceil(q / 256 c) quads into its accumulator; then come 5 warp-shuffle additions, 8 in the
CTA's sum of its warps and c in the last CTA's sum of the CTA partials.  A square therefore passes through at most
d = 4 k + 13 + c additions, and for non-negative terms each addition adds at most 2^-53 of the running sum, so the
partial is within d 2^-53 (1 + d 2^-53) of the exact sum.  The longest chain the tests meet is the canonical learner's
head segment at W = 1 (q = 1 697 728, c = 64, k = 104): d = 493, 5.5e-14.  numpy's pairwise float64 sum of the
reference adds less than 2^-53 * 64 of it.  1e-12 sits 18x above both, and far below what a dropped or doubled quad
changes."""
import ctypes as C
import math

import numpy as np
import torch

import adam_ref as AR
import head_ref as R
from helpers import assert_bits_equal

GUARD = 64                    # NaN floats after every param, grad and shard buffer
FLAG_NORM, FLAG_PARAM = 2, 3  # flag blocks of csrc/rb_peer.cu: [0] / [1] segment s reduced, [2] norm published, [3] parts stored
# The scratch layout of csrc/rb_peer.cu: PEER_SEGS (2) blocks of PEER_MAX_CTAS (592) double CTA partials, then double
# seg_norm[PEER_SEGS], then the unsigned tickets of the reduce of segment 0, of segment 1 and of k_peer_adam.
SEG_NORM_AT = 2 * 592                    # in doubles
TICKETS_AT = 2 * (SEG_NORM_AT + 2)       # in uint32
N_TICKETS = 3
SEG_NORM_RTOL = 1e-12

HYPER = (1.0, 1e-3, (0.9, 0.999), 1.5e-4)            # max_norm, lr, betas, eps
# the gradients of steps 1, 2, ...: a reduced norm far above max_norm, far below it, and all zero (coef = 1)
STEP_KINDS = ("clip", "noclip", "zero", "clip", "noclip")


def step_grad(seed, t, rank, numel, kind):
    """Rank `rank`'s float32 gradient at step t.  Independent normal draws of norm ~30 (clip) or ~0.01 (noclip) per rank,
    so the reduced norm is ~30 / sqrt(W) >= 10 or ~0.01 / sqrt(W) against max_norm 1."""
    if kind == "zero":
        return np.zeros(numel, dtype=np.float32)
    g = np.random.default_rng([seed, t, rank]).standard_normal(numel, dtype=np.float32)
    return g * np.float32((30.0 if kind == "clip" else 0.01) / math.sqrt(numel))


def learner_segments(arch):
    """The learner's flat layout and segments, built as FusedClipAdam builds them (on the host): segment 0 is the noisy
    head [conv_end, numel), reduced first; segment 1 the conv body [0, conv_end)."""
    from rainbow_b200.agent import FusedClipAdam
    from rainbow_b200.model import DQN
    from test_cpu_host import make_args
    hidden = {"canonical": 512, "data-efficient": 256}[arch]
    opt = FusedClipAdam(DQN(make_args(architecture=arch, hidden_size=hidden), 6), lr=1e-4, eps=1e-4, max_norm=10.0)
    return [(opt.conv_end, opt.numel), (0, opt.conv_end)]


def shard_slices(segments, world, rank):
    """[(flat slice owned by `rank`, slice inside its shard arrays)] per segment (PeerOptimizerState.shard_slices)."""
    out, off = [], 0
    for b, e in segments:
        part = (e - b) // world
        out.append((slice(b + rank * part, b + (rank + 1) * part), slice(off, off + part)))
        off += part
    return out


def reduced_grad(grads):
    """fl32(((0 + g_0) + g_1) + ...) * fl32(1/W), elementwise in float32, ranks in order."""
    acc = np.zeros_like(grads[0], dtype=np.float32)
    for g in grads:
        acc = acc + g
    return acc * np.float32(1.0 / len(grads))


def published_partial(seg_norm, n_seg):
    """What k_peer_adam publishes as its rank's share of the squared norm: 0.0 + seg_norm[0] (+ seg_norm[1])."""
    mine = 0.0
    for s in range(n_seg):
        mine += float(seg_norm[s])
    return mine


def flat_from_shards(snaps, segments, key):
    """The flat array (numel = segments' cover) whose owned slices are every rank's shard of `key`."""
    world = len(snaps)
    out = np.full(max(e for _, e in segments), np.nan, dtype=snaps[0][key].dtype)
    for r, s in enumerate(snaps):
        for fl, sh in shard_slices(segments, world, r):
            out[fl] = s[key][sh]
    return out


class World:
    """W emulated ranks of a P-element flat buffer cut into `segments` ([(begin, end)], at most two), on `device`."""

    def __init__(self, world, segments, device, lib):
        self.W, self.segments, self.lib = world, list(segments), lib
        self.P = max(e for _, e in segments)
        self.parts = [(e - b) // world for b, e in segments]
        self.shard = sum(self.parts)
        f32, f64, i64 = torch.float32, torch.float64, torch.int64

        def guarded(n, fill):
            t = torch.full((n + GUARD,), float("nan"), dtype=f32, device=device)
            t[:n].fill_(fill)
            return t

        self.ranks = [dict(param=guarded(self.P, float("nan")), grad=guarded(self.P, float("nan")),
                           flags=torch.zeros(4 * world, dtype=i64, device=device), norms=torch.zeros(world, dtype=f64, device=device),
                           gred=guarded(self.shard, float("nan")), exp_avg=guarded(self.shard, 0.0),
                           exp_avg_sq=guarded(self.shard, 0.0), step_count=torch.zeros(1, dtype=i64, device=device),
                           epoch=torch.zeros(1, dtype=i64, device=device), grad_norm=torch.full((1,), float("nan"), device=device),
                           scratch=torch.zeros(lib.rb_peer_scratch_bytes(), dtype=torch.uint8, device=device))
                      for _ in range(world)]
        ptrs = lambda key: (C.c_void_p * world)(*[rk[key].data_ptr() for rk in self.ranks])
        self.peer_param, self.peer_grad, self.peer_flags, self.peer_norms = (ptrs(k) for k in ("param", "grad", "flags", "norms"))
        self.seg_begin = (C.c_int64 * len(segments))(*[b for b, _ in segments])
        self.seg_len = (C.c_int64 * len(segments))(*[e - b for b, e in segments])
        self.launched = {}
        torch.cuda.synchronize(device)

    # -- the other ranks' part of the protocol -------------------------------------------------------------------------
    def begin_step(self):
        self.launched = {}

    def _emulate(self, r, groups):
        """groups: [(phase, flag blocks the launch waits on, whether it reads the norm slots)].  Publishes for every rank
        q != r that has not launched `phase` yet in this step, then checks every slot the launch waits on."""
        rk = self.ranks[r]
        e = int(rk["epoch"].item()) + 1
        for phase, blocks, norms in groups:
            for q in range(self.W):
                if q == r or q in self.launched.get(phase, ()):
                    continue
                for b in blocks:
                    rk["flags"][b * self.W + q] = e
                if norms:
                    assert all(q in self.launched.get(("reduce", s), ()) for s in range(len(self.segments))), \
                        f"emulation: rank {q}'s partial norm is read before it has reduced every segment"
                    rk["norms"][q] = self.partial(q)
        flags = rk["flags"].cpu().tolist()
        for _, blocks, _ in groups:
            for b in blocks:
                for q in range(self.W):
                    assert q == r or flags[b * self.W + q] >= e, \
                        f"rank {r} would wait on flag block {b} slot {q} = {flags[b * self.W + q]} < epoch {e}"

    def _mark_launched(self, r, *phases):
        for ph in phases:
            self.launched.setdefault(ph, set()).add(r)

    def seg_norm(self, r):
        return self.ranks[r]["scratch"].view(torch.float64)[SEG_NORM_AT:SEG_NORM_AT + 2].cpu().numpy()

    def partial(self, q):
        return published_partial(self.seg_norm(q), len(self.segments))

    # -- launches --------------------------------------------------------------------------------------------------------
    def _p(self, r, key, off=0):
        return self.ranks[r][key].data_ptr() + 4 * off

    def reduce(self, r, s, stream):
        from rainbow_b200 import _lib
        self._emulate(r, [(("reduce", s), (s,), False)])
        b, e = self.segments[s]
        _lib.check(self.lib.rb_peer_reduce(self.peer_grad, self.peer_flags, self.W, r, s, b, e - b, 1.0 / self.W,
                                           self._p(r, "gred", sum(self.parts[:s])), self._p(r, "epoch"), self._p(r, "scratch"),
                                           stream.cuda_stream))
        self._mark_launched(r, ("reduce", s))

    def prepare_adam(self, r):
        """The emulation for rank r's rb_peer_adam_gather (no launch)."""
        self._emulate(r, [("adam", (FLAG_NORM, FLAG_PARAM), True)])

    def launch_adam(self, r, hyper, stream):
        from rainbow_b200 import _lib
        max_norm, lr, (b1, b2), eps = hyper
        _lib.check(self.lib.rb_peer_adam_gather(
            self.peer_param, self.peer_flags, self.peer_norms, self.W, r, len(self.segments), self.seg_begin, self.seg_len,
            self._p(r, "gred"), self._p(r, "exp_avg"), self._p(r, "exp_avg_sq"), max_norm, lr, b1, b2, eps,
            self._p(r, "step_count"), self._p(r, "epoch"), self._p(r, "scratch"), self._p(r, "grad_norm"), None,
            stream.cuda_stream))
        self._mark_launched(r, "adam")

    def clip_adam(self, r, hyper, stream):
        """rb_peer_clip_adam: the one-segment reduce + adam_gather in one call."""
        from rainbow_b200 import _lib
        assert len(self.segments) == 1 and self.segments[0] == (0, self.P)
        self._emulate(r, [(("reduce", 0), (0,), False), ("adam", (FLAG_NORM, FLAG_PARAM), True)])
        max_norm, lr, (b1, b2), eps = hyper
        _lib.check(self.lib.rb_peer_clip_adam(
            self.peer_grad, self.peer_param, self.peer_flags, self.peer_norms, self.W, r, self.P, self._p(r, "gred"),
            self._p(r, "exp_avg"), self._p(r, "exp_avg_sq"), 1.0 / self.W, max_norm, lr, b1, b2, eps,
            self._p(r, "step_count"), self._p(r, "epoch"), self._p(r, "scratch"), self._p(r, "grad_norm"), stream.cuda_stream))
        self._mark_launched(r, ("reduce", 0), "adam")

    def reduce_all(self, side):
        """Starts a step of a two-segment world: every rank reduces segment 0 on `side`, then segment 1."""
        cur = torch.cuda.current_stream()
        self.begin_step()
        for r in range(self.W):
            side.wait_stream(cur)
            self.reduce(r, 0, side)
            cur.wait_stream(side)
            self.reduce(r, 1, cur)
            torch.cuda.synchronize()

    def step(self, hyper, side):
        """One optimiser step of every rank, in rank order, synchronising after each launch.  Two segments: like the
        learner, segment 0 is reduced on the side stream `side`, segment 1 after it on the current stream, then the
        norm exchange + Adam + all-gather.  One segment: rb_peer_clip_adam; ranks 1.. reduce once beforehand so that
        the partial norms rank 0's launch reads exist (the reduce is deterministic: the wrapper's second reduce rewrites
        the same gred and seg_norm, and the checks after the step would see it if it did not)."""
        cur = torch.cuda.current_stream()
        if len(self.segments) == 1:
            self.begin_step()
            for r in range(1, self.W):
                self.reduce(r, 0, cur)
                torch.cuda.synchronize()
            for r in range(self.W):
                self.clip_adam(r, hyper, cur)
                torch.cuda.synchronize()
            return
        self.reduce_all(side)
        for r in range(self.W):
            self.prepare_adam(r)
            self.launch_adam(r, hyper, cur)
            torch.cuda.synchronize()

    # -- state ------------------------------------------------------------------------------------------------------------
    def snapshot(self):
        """Host copies of every rank's state, in the form check_step reads."""
        out = []
        for rk in self.ranks:
            sc = rk["scratch"]
            out.append(dict(
                param=rk["param"][:self.P].cpu().numpy(), gred=rk["gred"][:self.shard].cpu().numpy(),
                exp_avg=rk["exp_avg"][:self.shard].cpu().numpy(), exp_avg_sq=rk["exp_avg_sq"][:self.shard].cpu().numpy(),
                step_count=int(rk["step_count"].item()), epoch=int(rk["epoch"].item()), grad_norm=rk["grad_norm"].cpu().numpy(),
                norms=rk["norms"].cpu().numpy(), flags=rk["flags"].cpu().numpy(),
                seg_norm=sc.view(torch.float64)[SEG_NORM_AT:SEG_NORM_AT + 2].cpu().numpy(),
                tickets=sc.view(torch.int32)[TICKETS_AT:TICKETS_AT + N_TICKETS].cpu().numpy(),
                guards={k: rk[k][-GUARD:].cpu().numpy() for k in ("param", "grad", "gred", "exp_avg", "exp_avg_sq")}))
        return out

    def state(self):
        return [{k: v.clone() for k, v in rk.items()} for rk in self.ranks]

    def restore(self, state):
        for rk, st in zip(self.ranks, state):
            for k, v in st.items():
                rk[k].copy_(v)
        torch.cuda.synchronize()


def check_step(snaps, before, grads, segments, t, hyper, device):
    """Every check after step t (1-based) of a world whose per-rank states are `snaps` (World.snapshot() or the same
    fields gathered from real ranks), from the state `before` the step and the ranks' gradients `grads` (float32 numpy).
    Returns the reference clip coefficient."""
    W, n_seg = len(snaps), len(segments)
    max_norm, lr, (b1, b2), eps = hyper
    for r, s in enumerate(snaps):
        assert s["step_count"] == t and s["epoch"] == t, f"rank {r}: step_count {s['step_count']}, epoch {s['epoch']} after step {t}"
        for k, g in s.get("guards", {}).items():
            assert np.isnan(g).all(), f"rank {r}: the guard after {k} was written"
        assert not s["tickets"].any(), f"rank {r}: tickets {s['tickets']} not back to 0"
        blocks = list(range(n_seg)) + [FLAG_NORM, FLAG_PARAM]
        flags = s["flags"].reshape(4, W)
        for b in range(4):
            want = t if b in blocks else 0
            assert (flags[b] == want).all(), f"rank {r}: flag block {b} = {flags[b].tolist()}, expected {want}"
    # gred: bitwise, from the gradients
    ref_g = reduced_grad(grads)
    for r, s in enumerate(snaps):
        for fl, sh in shard_slices(segments, W, r):
            assert_bits_equal(s["gred"][sh], ref_g[fl], f"rank {r} gred of flat {fl.start}:{fl.stop}")
    # seg_norm: float64 sum of squares of the kernel's own gred part
    for r, s in enumerate(snaps):
        for k, (fl, sh) in enumerate(shard_slices(segments, W, r)):
            ref = float(np.square(s["gred"][sh].astype(np.float64)).sum())
            got = float(s["seg_norm"][k])
            assert abs(got - ref) <= SEG_NORM_RTOL * ref, f"rank {r} seg_norm[{k}] {got!r} vs float64 {ref!r}"
    # the norm exchange: published partials, then one bitwise norm everywhere
    partials = [published_partial(s["seg_norm"], n_seg) for s in snaps]
    for r, s in enumerate(snaps):
        for q in range(W):
            assert_bits_equal(s["norms"][q:q + 1], np.array([partials[q]]), f"rank {r} norm slot {q}")
        n2 = 0.0
        for q in range(W):
            n2 += float(s["norms"][q])
        assert_bits_equal(s["grad_norm"], np.array([math.sqrt(n2)], dtype=np.float32), f"rank {r} grad_norm")
        assert_bits_equal(s["grad_norm"], snaps[0]["grad_norm"], f"rank {r} grad_norm vs rank 0")
        assert_bits_equal(s["param"], snaps[0]["param"], f"rank {r} parameters vs rank 0")
    # clip + Adam from the kernel's gred and the moments before the step
    tt = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    g = tt(flat_from_shards(snaps, segments, "gred"))
    m0, v0 = (tt(flat_from_shards(before, segments, k)) for k in ("exp_avg", "exp_avg_sq"))
    ref = AR.clip_adam(tt(before[0]["param"]), g, m0, v0, t - 1, 1.0, max_norm, lr, b1, b2, eps)
    R.assert_within("grad_norm", tt(snaps[0]["grad_norm"]), torch.tensor([ref["norm"][0]], dtype=torch.float64, device=device),
                    torch.tensor([ref["norm"][1]], dtype=torch.float64, device=device), AR.TAU)
    for name, got in (("m", tt(flat_from_shards(snaps, segments, "exp_avg"))), ("v", tt(flat_from_shards(snaps, segments, "exp_avg_sq"))),
                      ("p", tt(snaps[0]["param"]))):
        val, scale = ref[name]
        R.assert_within(f"{name} after step {t}", got, val, scale, AR.TAU)
    return ref["coef"]
