"""Peer-memory optimiser state for multi-GPU learners (NVLink / NVSwitch, one process per GPU).

Design (SURVEY.md 8(e); brief: "where a hot op is a compute step followed by a collective, write ONE kernel that does both
over peer memory"): the flat gradient and parameter buffers of every rank live in symmetric memory mapped on all GPUs.
Per update (csrc/rb_peer.cu)
  1. `reduce_segment(0)`: reduce-scatter of the noisy-head segment of the gradient with peer LOADS, enqueued on a side
     stream as soon as the head backward is done, so it crosses NVLink while the conv backward is still running;
  2. `step()`: reduce-scatter of the (small) conv segment, exchange of the partial norms, clip + Adam on the owned 1/world
     parts only -- the Adam moments are sharded --, all-gather of the updated parameters with peer STORES;
cross-GPU ordering is epoch flags in the same symmetric allocation, never the host.  Replaces
`all_reduce(flat_grad); rb_clip_adam` (replicated 192 MB optimiser pass on every rank).

tests/test_gpu_peer_f64.py checks every stage against a float64 reference with W = 1, 2, 4 and 8 ranks emulated on one
GPU, and this class over real symmetric memory on a host with 2+ GPUs; tools/peer_adam_check.py compares it against the
NCCL path on a multi-GPU node.  `args.peer_optimizer`: True | "auto" (falls back to the NCCL all-reduce when symmetric
memory cannot be set up; bench.py's default for world > 1) | False.
"""
import ctypes as C

import torch
import torch.distributed as dist

from . import _lib

_KEEP = []   # symmetric-memory handles must outlive every kernel that uses the peer mappings


def _peer_allocate(total_bytes, device, group):
    """A zeroed `total_bytes` uint8 buffer on `device` that every rank of `group` can address (torch symmetric memory:
    cuMem allocation + handle exchange): returns (local tensor, [base pointer of every rank's buffer as seen from here])."""
    import os
    if os.environ.get("RB_PEER_MULTICAST", "0") != "1":
        # the NVSwitch multicast mapping is not used by default, so torch is told not to create one: multicast-group creation
        # goes through the fabric manager, the step the round-1 communicator hang sat in (DESIGN.md 6)
        os.environ.setdefault("TORCH_SYMM_MEM_DISABLE_MULTICAST", "1")
    import torch.distributed._symmetric_memory as symm_mem
    grp = group if group is not None else dist.group.WORLD
    buf = symm_mem.empty(total_bytes, dtype=torch.uint8, device=device)
    buf.zero_()
    handle = symm_mem.rendezvous(buf, grp.group_name)
    _KEEP.append(handle)
    mc = 0
    try:   # NVLS multicast mapping of the same allocation (0 when the fabric / driver does not offer it)
        mc = int(handle.multicast_ptr or 0)
    except Exception:
        mc = 0
    return buf, [int(p) for p in handle.buffer_ptrs], mc


class PeerOptimizerState:
    """Symmetric allocation holding [flat_param | flat_grad | flags | norms] of one rank, rendezvoused over `group`.

    `segments`: [(begin, end), ...] (at most two) covering [0, numel): the order in which the gradient becomes final.
    Segment 0 may be reduced early with reduce_segment(0); step() reduces whatever is left."""

    def __init__(self, numel, device, segments=None, group=None):
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        if self.world not in (2, 4, 8):
            raise _lib.RainbowB200Error("peer optimiser supports 2, 4 or 8 ranks (one NVLink domain)")
        q = 4 * self.world
        if numel % q:
            raise _lib.RainbowB200Error(f"flat buffer length {numel} is not a multiple of 4 * world")
        self.numel = numel
        segments = [(0, numel)] if segments is None else [s for s in segments if s[1] > s[0]]
        if not 1 <= len(segments) <= 2 or sorted(segments)[0][0] != 0 or sorted(segments)[-1][1] != numel:
            raise _lib.RainbowB200Error("segments must be one or two ranges covering the flat buffer")
        for b, e in segments:
            if b % 4 or (e - b) % q:
                raise _lib.RainbowB200Error("every segment must start on a multiple of 4 and hold a multiple of 4 * world elements")
        self.segments = segments
        self.parts = [(e - b) // self.world for b, e in segments]
        self.shard = sum(self.parts)
        pbytes = numel * 4
        fbytes = 4 * self.world * 8
        nbytes = self.world * 8
        self._off = (0, pbytes, 2 * pbytes, 2 * pbytes + 256 * (-(-fbytes // 256)))
        total = self._off[3] + 256 * (-(-nbytes // 256))
        self.buf, bases, mc = _peer_allocate(total, device, group)
        import os
        # RB_PEER_MULTICAST=1: the parameter all-gather goes through the NVSwitch multicast mapping (one multimem.st per 16
        # bytes instead of `world` peer stores).  Validated (tools/peer_adam_check.py) but not faster at N = 2 (mgpu_q2:
        # k_peer_adam 70 us vs 44 us with peer stores), so it is opt-in until it has been measured at N = 8.
        self.multicast = bool(mc) and os.environ.get("RB_PEER_MULTICAST", "0") == "1"
        self._mc_param = C.c_void_p(mc + self._off[0]) if self.multicast else None
        self.flat_param = self.buf[self._off[0]:self._off[0] + pbytes].view(torch.float32)
        self.flat_grad = self.buf[self._off[1]:self._off[1] + pbytes].view(torch.float32)
        n = self.world
        self._peer_param = (C.c_void_p * n)(*[b + self._off[0] for b in bases])
        self._peer_grad = (C.c_void_p * n)(*[b + self._off[1] for b in bases])
        self._peer_flags = (C.c_void_p * n)(*[b + self._off[2] for b in bases])
        self._peer_norms = (C.c_void_p * n)(*[b + self._off[3] for b in bases])
        self._seg_begin = (C.c_int64 * len(segments))(*[b for b, _ in segments])
        self._seg_len = (C.c_int64 * len(segments))(*[e - b for b, e in segments])
        f32 = torch.float32
        self.gred = torch.zeros(self.shard, dtype=f32, device=device)
        self.exp_avg = torch.zeros(self.shard, dtype=f32, device=device)      # this rank's shard of the moments
        self.exp_avg_sq = torch.zeros(self.shard, dtype=f32, device=device)
        self.step_count = torch.zeros(1, dtype=torch.int64, device=device)
        self.epoch = torch.zeros(1, dtype=torch.int64, device=device)
        self.grad_norm = torch.zeros(1, dtype=f32, device=device)
        self._lib = _lib.load()
        self._scratch = torch.zeros(self._lib.rb_peer_scratch_bytes(), dtype=torch.uint8, device=device)
        self._reduced = [False] * len(segments)
        torch.cuda.synchronize(device)
        dist.barrier(group)                                   # every rank's zeroed flags are in place before the first step

    def shard_slices(self):
        """[(flat slice owned by this rank, slice inside the shard arrays)] per segment."""
        out, off = [], 0
        for (b, _), part in zip(self.segments, self.parts):
            out.append((slice(b + self.rank * part, b + (self.rank + 1) * part), slice(off, off + part)))
            off += part
        return out

    def reduce_segment(self, s):
        """Reduce-scatter of segment `s` on the current stream (its gradients must be final in stream order)."""
        b, e = self.segments[s]
        off = sum(self.parts[:s])
        _lib.check(self._lib.rb_peer_reduce(
            self._peer_grad, self._peer_flags, self.world, self.rank, s, b, e - b, 1.0 / self.world,
            _lib.ptr(self.gred[off:off + self.parts[s]]), _lib.ptr(self.epoch), _lib.ptr(self._scratch), _lib.stream()))
        self._reduced[s] = True

    def step(self, max_norm, lr, betas, eps, weight_decay=None, seg_steps=None):
        """`seg_steps` (device int64[segments], each segment's own bias-correction count): AdamW with decoupled decay
        `weight_decay` on every segment (rb_peer_adamw_gather); None: plain Adam (rb_peer_adam_gather)."""
        for s in range(len(self.segments)):
            if not self._reduced[s]:
                self.reduce_segment(s)
        if seg_steps is not None:
            n = len(self.segments)
            _lib.check(self._lib.rb_peer_adamw_gather(
                self._peer_param, self._peer_flags, self._peer_norms, self.world, self.rank, n, self._seg_begin,
                self._seg_len, (C.c_float * n)(*([float(weight_decay or 0.0)] * n)), _lib.ptr(self.gred),
                _lib.ptr(self.exp_avg), _lib.ptr(self.exp_avg_sq), float(max_norm), float(lr), float(betas[0]),
                float(betas[1]), float(eps), _lib.ptr(self.step_count), _lib.ptr(seg_steps), _lib.ptr(self.epoch),
                _lib.ptr(self._scratch), _lib.ptr(self.grad_norm), self._mc_param, _lib.stream()))
        else:
            _lib.check(self._lib.rb_peer_adam_gather(
                self._peer_param, self._peer_flags, self._peer_norms, self.world, self.rank, len(self.segments),
                self._seg_begin, self._seg_len, _lib.ptr(self.gred), _lib.ptr(self.exp_avg), _lib.ptr(self.exp_avg_sq),
                float(max_norm), float(lr), float(betas[0]), float(betas[1]), float(eps), _lib.ptr(self.step_count),
                _lib.ptr(self.epoch), _lib.ptr(self._scratch), _lib.ptr(self.grad_norm), self._mc_param, _lib.stream()))
        self._reduced = [False] * len(self.segments)
