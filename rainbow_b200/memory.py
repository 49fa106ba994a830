"""Prioritised replay living entirely in GPU HBM.

Mirrors the class surface of the reference's memory.py (SegmentTree memory.py:12-89, ReplayMemory
memory.py:91-180) so main.py / test.py / agent.py of the reference run against it unchanged, but the
state is a structure of arrays on the device and every operation is one hand-written CUDA kernel
called through the C ABI in include/rainbow_b200.h:

    append             -> rb_append        (K5)   memory.py:105-108, 56-61
    append_truncated   -> rb_append_batch_trunc   (args.bootstrap_truncation: a time limit's last step and the
                                                   observation it stopped at, no reference counterpart)
    sample             -> rb_tree_sample   (K1)   memory.py:124-132, 148-154
                          rb_gather        (K2)   memory.py:111-121, 134-146
                          (rb_gather_shift with shift_pad > 0: the same plus random-shift augmentation, no reference
                          counterpart; rb_gather_aug with intensity > 0 or copies != (1, 1): shift and intensity
                          augmentation of M copies of s and K of s'; rb_gather_horizon with an annealed horizon, see
                          rainbow_b200.horizon; rb_gather_trunc with args.bootstrap_truncation)
    extend             -> rb_append_bulk          (k appends of quantised arrays in one call: a dataset fill, no
                                                   reference counterpart)
    update_priorities  -> rb_tree_update   (K4)   memory.py:157-159, 23-48
    __next__           -> rb_iter_states          memory.py:166-178

HBM layout (per ReplayMemory): float32 sum tree [tree_start+size] in heap order (one pad float in
front so level runs are 128-byte aligned), uint8 frames [size,7056], int32 timestep/action,
float32 reward, uint8 nonterminal: 7069 B per transition like the reference's packed record, i.e.
7.07 GB at the default 1M capacity.

Randomness: `rng="philox"` (default) draws the stratified uniforms on the device (Philox4x32-10,
counter kept on the device so CUDA-graph replays advance it); `rng="numpy"` consumes the global
legacy numpy generator exactly like memory.py:129 does, which makes sampled indices bit-identical to
the reference for the same seed and tree (at the price of one small H2D copy and a status read).
"""
import numpy as np
import torch

from . import _lib

FRAME = 84 * 84
FINAL = 2   # RB_NONTERMINAL_FINAL: the nonterminal byte of a final-observation record (append_truncated)

# memory.py:7 -- only used to exchange state with reference-format consumers (pickles)
Transition_dtype = np.dtype([("timestep", np.int32), ("state", np.uint8, (84, 84)), ("action", np.int32),
                             ("reward", np.float32), ("nonterminal", np.bool_)])
Final_transition_dtype = np.dtype(Transition_dtype.descr + [("final", np.bool_)])


# The replay's persistent fields, one list for pickling (ReplayMemory.__getstate__ / __setstate__) and for
# rainbow_b200.checkpoint: host attributes of the ReplayMemory with their role on a checkpoint restore -- "structure" must
# match the live object, "setting" keeps the live object's value, "state" is restored -- and the device arrays of its
# SegmentTree as (pickle key, SegmentTree attribute).  Both formats add the ring's host mirrors (index, full) and device
# scalars (running max, sampling counter) in their own form.
PERSISTENT_ROLES = (("capacity", "structure"), ("history", "structure"), ("discount", "setting"), ("n", "setting"),
                    ("priority_weight", "state"), ("priority_exponent", "setting"), ("t", "state"), ("rng", "setting"),
                    ("seed", "state"), ("max_attempts", "setting"), ("strict", "setting"))
PERSISTENT_HOST = tuple(name for name, _ in PERSISTENT_ROLES)
PERSISTENT_ARRAYS = (("sum_tree", "tree"), ("frames", "frames"), ("timestep", "timestep"), ("action", "action"),
                     ("reward", "reward"), ("nonterminal", "nonterminal"))


def _require_cuda(device):
    device = torch.device(device)
    if device.type != "cuda":
        raise _lib.RainbowB200Error(
            f"rainbow_b200.ReplayMemory needs a CUDA device, got '{device}': the replay lives in HBM and there "
            "is no CPU fallback")
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    return device


class SegmentTree:
    """Device-resident counterpart of memory.py:12-89.  `index`, `full`, `size`, `tree_start` are host
    mirrors (cheap ints, advanced in lock step with the device copy in `ring_state`); `max`, `sum_tree`
    and `data` read the device and therefore synchronise -- they exist for inspection and pickling."""

    def __init__(self, size, device):
        size = int(size)
        if size <= 0 or size % 2:
            # the reference itself raises IndexError in _propagate_index for odd sizes (SURVEY.md App. A.1)
            raise ValueError("SegmentTree size must be a positive even number")
        self.device = _require_cuda(device)
        self.size = size
        self.tree_start = 2 ** (size - 1).bit_length() - 1
        self.index = 0
        self.full = False
        n = self.tree_start + size
        # one pad element in front: node j lives at element j+1, so the 32-node run of a tree level starts
        # on a 128-byte boundary
        self._tree_store = torch.zeros(n + 1, dtype=torch.float32, device=self.device)
        self.tree = self._tree_store[1:]
        self.frames = torch.zeros((size, FRAME), dtype=torch.uint8, device=self.device)
        self.timestep = torch.zeros(size, dtype=torch.int32, device=self.device)
        self.action = torch.zeros(size, dtype=torch.int32, device=self.device)
        self.reward = torch.zeros(size, dtype=torch.float32, device=self.device)
        self.nonterminal = torch.zeros(size, dtype=torch.uint8, device=self.device)
        self.final_records = False   # get() adds a `final` field (ReplayMemory with args.bootstrap_truncation)
        self.ring_state = torch.zeros(5, dtype=torch.int64, device=self.device)  # head, full, t_episode, appended, ticket
        self.running_max = torch.ones(1, dtype=torch.float32, device=self.device)  # memory.py:20
        self._status = torch.zeros(4, dtype=torch.int32, device=self.device)
        self._lib = _lib.load()

    # ---- pickling: the reference pickles the whole object graph (main.py:85-100) ------------------------------
    def __getstate__(self):
        """The reference's own field layout (memory.py:13-20): index, size, full, tree_start, sum_tree, data, max."""
        return dict(index=self.index, size=self.size, full=self.full, tree_start=self.tree_start, sum_tree=self.sum_tree,
                    data=self.data, max=self.max)

    def __setstate__(self, state):
        """Accepts the reference's SegmentTree.__dict__ (a file written by the reference, loaded with dropin/ shadowing
        the `memory` module).  The device arrays are created by _materialise() once the owning ReplayMemory knows the device."""
        if not all(k in state for k in ("index", "size", "full", "sum_tree", "data", "max")):
            raise _lib.RainbowB200Error("unknown SegmentTree pickle layout")
        self._pending = dict(state)
        self.size, self.index, self.full = int(state["size"]), int(state["index"]), bool(state["full"])
        self.tree_start = 2 ** (self.size - 1).bit_length() - 1

    def _materialise(self, device, t_episode=0):
        fields = self.__dict__.pop("_pending")
        SegmentTree.__init__(self, fields["size"], device)
        self.load_arrays(**reference_fields_to_ring(fields, t=t_episode))

    # ---- reference-style accessors -------------------------------------------------------------
    @property
    def max(self):
        return float(self.running_max.item())

    @property
    def sum_tree(self):
        return self.tree.cpu().numpy()

    @property
    def data(self):
        out = np.zeros(self.size, dtype=Transition_dtype)
        out["timestep"] = self.timestep.cpu().numpy()
        out["state"] = self.frames.cpu().numpy().reshape(self.size, 84, 84)
        out["action"] = self.action.cpu().numpy()
        out["reward"] = self.reward.cpu().numpy()
        out["nonterminal"] = self.nonterminal.cpu().numpy().astype(np.bool_)
        return out

    def total(self):
        return self.tree[0].item()

    # ---- operations ----------------------------------------------------------------------------
    def _as_dev(self, x, dtype):
        if isinstance(x, torch.Tensor):
            return x.to(device=self.device, dtype=dtype).contiguous()
        return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype).to(self.device, non_blocking=True)

    def update(self, indices, values, omega=None, gate=None):
        """memory.py:44-48.  `values` are tree values; with `omega` given they are raw priorities and the
        kernel applies ^omega (memory.py:158).  `gate`: optional device int32 tensor; the launch is a no-op when its
        first element is 0 (the status word of a rejected sample batch)."""
        idx = self._as_dev(indices, torch.int64).reshape(-1)
        val = self._as_dev(values, torch.float32).reshape(-1)
        if idx.numel() != val.numel():
            raise ValueError("indices and values differ in length")
        _lib.check(self._lib.rb_tree_update(
            _lib.ptr(self.tree), self.tree_start, self.size, _lib.ptr(idx), _lib.ptr(val),
            0.0 if omega is None else float(omega), 1 if omega is None else 0, idx.numel(),
            _lib.ptr(self.running_max), _lib.ptr(self._status), _lib.ptr(gate), _lib.stream()))

    def find(self, values):
        """memory.py:79-82: float64 values -> (leaf values, data indices, tree indices), as device tensors."""
        v = self._as_dev(values, torch.float64).reshape(-1)
        B = v.numel()
        probs = torch.empty(B, dtype=torch.float32, device=self.device)
        didx = torch.empty(B, dtype=torch.int64, device=self.device)
        tidx = torch.empty(B, dtype=torch.int64, device=self.device)
        _lib.check(self._lib.rb_tree_find(_lib.ptr(self.tree), self.tree_start, self.size, _lib.ptr(v), B,
                                          _lib.ptr(probs), _lib.ptr(didx), _lib.ptr(tidx), _lib.stream()))
        return probs, didx, tidx

    def append_frame(self, last_frame, action, reward, terminal):
        """memory.py:56-61 with the record fields passed separately; the leaf gets the running max.
        `last_frame`: float32 [84*84] in device memory or PINNED host memory (read in place by the kernel)."""
        fptr = last_frame.data_ptr() if (not last_frame.is_cuda and last_frame.is_pinned()) else _lib.ptr(last_frame)
        _lib.check(self._lib.rb_append(
            _lib.ptr(self.tree), self.tree_start, self.size, _lib.ptr(self.frames), _lib.ptr(self.timestep),
            _lib.ptr(self.action), _lib.ptr(self.reward), _lib.ptr(self.nonterminal), _lib.ptr(self.ring_state),
            _lib.ptr(self.running_max), fptr, int(action), float(reward), 1 if terminal else 0,
            _lib.stream()))
        self.index = (self.index + 1) % self.size
        self.full = self.full or self.index == 0

    def get(self, data_index):
        """memory.py:85-86 (host copy of the selected records; inspection only).  With final_records set the records
        carry one more bool field, `final`: a final-observation record (whose `nonterminal` reads True)."""
        idx = np.asarray(data_index) % self.size
        flat = torch.as_tensor(idx.reshape(-1), dtype=torch.int64, device=self.device)
        dtype = Final_transition_dtype if self.final_records else Transition_dtype
        out = np.zeros(idx.size, dtype=dtype)
        out["timestep"] = self.timestep[flat].cpu().numpy()
        out["state"] = self.frames[flat].cpu().numpy().reshape(-1, 84, 84)
        out["action"] = self.action[flat].cpu().numpy()
        out["reward"] = self.reward[flat].cpu().numpy()
        nonterminal = self.nonterminal[flat].cpu().numpy()
        out["nonterminal"] = nonterminal.astype(np.bool_)
        if self.final_records:
            out["final"] = nonterminal == FINAL
        return out.reshape(idx.shape)

    # ---- bulk state exchange (tests, pickling, synthetic fill) -----------------------------------
    def load_arrays(self, sum_tree=None, frames=None, timestep=None, action=None, reward=None, nonterminal=None,
                    index=None, full=None, t_episode=0, max_value=None):
        def put(dst, src, dt):
            if src is not None:
                dst.copy_(torch.as_tensor(np.ascontiguousarray(src), dtype=dt).reshape(dst.shape))

        put(self.tree, sum_tree, torch.float32)
        put(self.frames, frames, torch.uint8)
        put(self.timestep, timestep, torch.int32)
        put(self.action, action, torch.int32)
        put(self.reward, reward, torch.float32)
        put(self.nonterminal, None if nonterminal is None else np.asarray(nonterminal).astype(np.uint8), torch.uint8)
        if index is not None:
            self.index = int(index)
        if full is not None:
            self.full = bool(full)
        self.ring_state.copy_(torch.tensor([self.index, int(self.full), int(t_episode), 0, 0], dtype=torch.int64))
        if max_value is not None:
            self.running_max.fill_(float(max_value))


class _SampleWorkspace:
    """Output buffers of one sample() call for a given batch size."""

    def __init__(self, B, history, device, copies=(1, 1)):
        f32, i64 = torch.float32, torch.int64
        self.B = B
        self.copies = M, K = (int(copies[0]), int(copies[1]))
        self.probs = torch.empty(B, dtype=f32, device=device)
        self.data_idx = torch.empty(B, dtype=i64, device=device)
        self.tree_idx = torch.empty(B, dtype=i64, device=device)
        self.weights = torch.empty(B, dtype=f32, device=device)
        # one allocation, s rows then s' rows: the learner can push [s; s'] through the online conv body in a single pass.
        # With copies = (M, K) (rb_gather_aug) it holds M copies of s, then K copies of s', copy-major: [(M + K) B] rows.
        self.both_states = torch.empty(((M + K) * B, history, 84, 84), dtype=f32, device=device)
        self.states, self.next_states = self.both_states[:M * B], self.both_states[M * B:]
        self.actions = torch.empty(B, dtype=i64, device=device)
        self.returns = torch.empty(B, dtype=f32, device=device)
        self.nonterminals = torch.empty((B, 1), dtype=f32, device=device)
        self.status = torch.zeros(4, dtype=torch.int32, device=device)   # ok flag, draws used, rejected batches so far, -
        self.shifts = None   # int32 [2][B][2] offsets of the last shifted gather, [2][max(M, K)][B][2] after rb_gather_aug
        self.scales = None   # float32 [2][max(M, K)][B] intensity multipliers of the last rb_gather_aug

    def as_tuple(self):
        return (self.tree_idx, self.states, self.actions, self.returns, self.next_states, self.nonterminals,
                self.weights)


class ReplayMemory:
    """Drop-in for memory.py:91-180 (`ReplayMemory(args, capacity)`).

    Extra keyword arguments (not in the reference): rng ("philox" | "numpy"), seed, max_attempts,
    strict (read the kernel's status word after every sample and raise if the batch was rejected
    max_attempts times -- costs a device synchronisation)."""

    APPEND_BATCH = 8  # RB_APPEND_BATCH
    MAX_SHIFT_PAD = 16  # RB_MAX_SHIFT_PAD
    MAX_AUG_COPIES = 8  # RB_MAX_AUG_COPIES
    MAX_INTENSITY = 0.5

    def __init__(self, args, capacity, rng="philox", seed=None, max_attempts=64, strict=False, defer_appends=False):
        self.device = _require_cuda(args.device)
        self.capacity = int(capacity)
        self.history = int(args.history_length)
        self.discount = args.discount
        self.n = int(args.multi_step)
        if getattr(args, "anneal_steps", None):   # an annealed horizon (rainbow_b200.horizon): the window of its longest n
            self.n = max(self.n, int(getattr(args, "multi_step_start", None) or self.n))
        self.priority_weight = args.priority_weight  # beta; main.py:161 overwrites this attribute every step
        self.priority_exponent = args.priority_exponent
        # bootstrapping through time limits: append_truncated stores the observation a time limit stopped the episode
        # at, and the gather cuts a sample's window there (rb_gather_trunc, nonterminals in discount form)
        self.bootstrap_truncation = bool(getattr(args, "bootstrap_truncation", False))
        if self.history + self.n > 64:
            raise ValueError("history_length + multi_step must not exceed 64")
        if rng not in ("philox", "numpy"):
            raise ValueError("rng must be 'philox' or 'numpy'")
        self.rng = rng
        self.max_attempts = int(max_attempts)
        self.strict = bool(strict)
        # defer_appends: append() only queues (frame reference + fields); the queue is written by ONE rb_append_batch
        # launch before the next read of the replay (sample / update_priorities / iteration / pickling) or when it holds
        # APPEND_BATCH transitions.  The caller must not modify a queued frame tensor before the flush.
        # [round-1 status: off by default, not yet exercised on hardware]
        self.defer_appends = bool(defer_appends)
        self._queue = []
        self.t = 0  # in-episode step of the next append (memory.py:100); device copy in ring_state[2]
        # memory.py:101: [gamma**i] in Python doubles, then float32
        self.n_step_scaling = torch.tensor([self.discount ** i for i in range(self.n)], dtype=torch.float32,
                                           device=self.device)
        self.transitions = SegmentTree(self.capacity, self.device)
        if self.bootstrap_truncation:
            self.transitions.final_records = True
        self._fixed_row = self._fixed_horizon_row()
        if seed is None:   # data-parallel ranks launched with one torch seed must not draw the same stratified uniforms
            from .dist import GradSync, shard_seed
            rank = GradSync().rank
            seed = torch.initial_seed() if rank == 0 else shard_seed(torch.initial_seed(), rank)
        self.seed = int(seed) & (2 ** 64 - 1)
        self._rng_counter = torch.zeros(1, dtype=torch.int64, device=self.device)
        self._beta_dev = torch.full((1,), float(self.priority_weight), dtype=torch.float32, device=self.device)
        self._beta_pushed = float(self.priority_weight)
        self._lib = _lib.load()
        self._last = None
        self._stage = None

    def _fixed_horizon_row(self):
        """With bootstrap_truncation: the constant rb_horizon row of this replay's n and discount that rb_gather_trunc
        reads when no annealed horizon is given -- n, fl32(gamma ** n) and fl32(gamma ** k) for k < n, in Python doubles
        like n_step_scaling.  None without it."""
        if not self.bootstrap_truncation:
            return None
        from .horizon import horizon_table
        row = horizon_table(1, self.n, self.n, self.discount, self.discount)[:1]
        return torch.from_numpy(row.view(np.uint8).copy()).to(self.device)

    def holds_final_records(self):
        """Synchronises.  Whether the ring holds a final-observation record (append_truncated)."""
        self.flush_appends()
        return bool((self.transitions.nonterminal == FINAL).any().item())

    def push_beta(self):
        """Mirror the host attribute `priority_weight` (main.py:161 rewrites it every step) into the device
        scalar the sampling kernel reads, so a captured CUDA graph sees the current beta."""
        b = float(self.priority_weight)
        if b != self._beta_pushed:
            self._beta_dev.fill_(b)
            self._beta_pushed = b

    # ---- append --------------------------------------------------------------------------------
    STAGE_SLOTS = 16   # owned pinned staging frames for host-resident states (2 x APPEND_BATCH)

    def _stage_host_frame(self, last):
        """Copy a HOST frame into an owned pinned slot and return the slot (float32 [84*84], 16-byte aligned).

        The reference copies the frame synchronously (memory.py:106); an asynchronous H2D copy straight from the caller's
        buffer would race with an env that rewrites its (pinned) frame buffer in place.  The slot is reused only after the
        kernel that consumed it has finished (event per slot), so the caller may do whatever it likes with `state` as
        soon as append() returns."""
        if self._stage is None:
            self._stage = torch.empty((self.STAGE_SLOTS, FRAME), dtype=torch.float32).pin_memory()
            self._stage_evt = [None] * self.STAGE_SLOTS
            self._stage_next = 0
        k = self._stage_next
        self._stage_next = (k + 1) % self.STAGE_SLOTS
        if self._stage_evt[k] is not None:
            self._stage_evt[k].synchronize()
            self._stage_evt[k] = None
        slot = self._stage[k]
        slot.view(84, 84).copy_(last)      # host memcpy (+ dtype conversion / de-striding if needed)
        return k, slot

    def _release_stage_slots(self, slots):
        if slots:
            evt = torch.cuda.Event()
            evt.record(torch.cuda.current_stream(self.device))
            for k in slots:
                self._stage_evt[k] = evt

    def _newest_frame(self, state):
        """(staging slot or None, the newest frame of `state` as a 16-byte aligned float32 frame the kernel reads)."""
        last = state[-1]
        if not last.is_cuda:
            return self._stage_host_frame(last)
        last = last.to(torch.float32).contiguous()
        if last.data_ptr() % 16:
            last = last.clone()
        return None, last

    def append(self, state, action, reward, terminal):
        """memory.py:105-108.  `state` is the float32 [history,84,84] frame stack in [0,1]; only the newest
        frame is stored (quantised to uint8 on the device).  Host frames are staged through owned pinned memory and read
        by the kernel in place (no separate H2D copy launch); device frames are read in place."""
        slot_id, last = self._newest_frame(state)
        if self.defer_appends:
            # queued by reference: a DEVICE frame must not be modified by the caller before the flush (main.py's env
            # builds a fresh state tensor every step); host frames are already copied into the staging ring
            self._queue.append((last, int(action), float(reward), bool(terminal), slot_id))
            tr = self.transitions
            tr.index = (tr.index + 1) % tr.size       # host mirrors advance now, the device copy at the flush
            tr.full = tr.full or tr.index == 0
            self.t = 0 if terminal else self.t + 1
            if len(self._queue) >= self.APPEND_BATCH:
                self.flush_appends()
            return
        self.transitions.append_frame(last, action, reward, terminal)
        if slot_id is not None:
            self._release_stage_slots([slot_id])
        self.t = 0 if terminal else self.t + 1

    def append_truncated(self, state, action, reward, final_state):
        """A time limit's last step (needs args.bootstrap_truncation): the transition (state, action, reward) with
        nonterminal 1, then a final-observation record F holding the newest frame of `final_state` -- the observation the
        time limit stopped the episode at.  F continues the episode's timesteps, has action 0, reward 0, leaf priority 0
        (it is never sampled, and the running max stays) and the nonterminal byte FINAL; the next append starts an
        episode.  A sample whose n-step window reaches F bootstraps from the stack ending at F, k < n steps on
        (rb_gather_trunc).  One rb_append_batch_trunc launch, or two queued records with defer_appends."""
        if not self.bootstrap_truncation:
            raise _lib.RainbowB200Error("append_truncated needs args.bootstrap_truncation = True: without it the replay "
                                        "cannot store the final observation a time limit stopped the episode at")
        slot_id, last = self._newest_frame(state)
        final_slot_id, final = self._newest_frame(final_state)
        records = [(last, int(action), float(reward), 0, slot_id), (final, 0, 0.0, FINAL, final_slot_id)]
        tr = self.transitions
        if self.defer_appends:
            if len(self._queue) + 2 > self.APPEND_BATCH:
                self.flush_appends()
            self._queue += records
        else:
            self._append_batch(records)
        tr.index = (tr.index + 2) % tr.size
        tr.full = tr.full or tr.index < 2
        self.t = 0
        if self.defer_appends and len(self._queue) >= self.APPEND_BATCH:
            self.flush_appends()

    # ---- bulk fill from arrays ------------------------------------------------------------------
    EXTEND_CHUNK_BYTES = 64 << 20   # frames per rb_append_bulk call and per pinned staging buffer (two of them)

    def extend(self, frames, actions, rewards, terminals, final=None):
        """Append k transitions given as arrays, bitwise as k calls of append() (and append_truncated() for the pairs
        `final` marks) would leave the replay: frames, records, the whole sum tree, the running max, the ring state and
        the host mirrors index, full and t.  With k > capacity only the last `capacity` records remain.

        frames: uint8 [k, 84, 84] or [k, 7056], the newest frame of each state already quantised, as datasets store it:
        numpy, a CPU tensor (pageable or pinned) or a CUDA tensor on this replay's device (read in stream order on the
        current stream).  Float frames are refused; append's rounding is q = (uint8)(int)fl32(f * 255).
        actions (integers that fit int32), rewards (rounded to fp32 as append rounds float(reward)), terminals: [k].
        final (optional, [k] bool, needs args.bootstrap_truncation): record j is the final observation of a time-limited
        episode, so records j - 1 and j are what append_truncated(state_{j-1}, a, r, final_state_j) writes.  Record j - 1
        must be in the same call, neither terminal nor final; record j must have terminal False, action 0 and reward 0.

        Everything is checked before anything is written, and a refused call writes nothing.  A non-empty defer_appends
        queue is written first.  Host frames go through two owned pinned buffers of EXTEND_CHUNK_BYTES (a host copy into
        one while the copy engine moves the other), so the caller may reuse its arrays as soon as this returns; the host
        waits only on those buffers' events."""
        fr, acts, rews, flags = self._check_extend(frames, actions, rewards, terminals, final)
        k = flags.size
        if k == 0:
            return
        self.flush_appends()
        tr = self.transitions
        chunk = max(1, min(tr.size, self.EXTEND_CHUNK_BYTES // FRAME))
        stage = self._extend_stage(min(chunk, k), fr.is_cuda)
        stream = torch.cuda.current_stream(self.device)
        for c, j0 in enumerate(range(0, k, chunk)):
            n = min(chunk, k - j0)
            b = c % 2
            if stage["evt"][b] is not None:
                stage["evt"][b].synchronize()
            stage["act"][b][:n].copy_(torch.from_numpy(acts[j0:j0 + n]))
            stage["rew"][b][:n].copy_(torch.from_numpy(rews[j0:j0 + n]))
            stage["flag"][b][:n].copy_(torch.from_numpy(flags[j0:j0 + n]))
            if fr.is_cuda:
                src = fr[j0:j0 + n]
            else:
                stage["frames"][b][:n].copy_(fr[j0:j0 + n])
                src = stage["frames"][b]
            dev = stage["dev"]
            dev["act"][:n].copy_(stage["act"][b][:n], non_blocking=True)
            dev["rew"][:n].copy_(stage["rew"][b][:n], non_blocking=True)
            dev["flag"][:n].copy_(stage["flag"][b][:n], non_blocking=True)
            _lib.check(self._lib.rb_append_bulk(
                _lib.ptr(tr.tree), tr.tree_start, tr.size, _lib.ptr(tr.frames), _lib.ptr(tr.timestep),
                _lib.ptr(tr.action), _lib.ptr(tr.reward), _lib.ptr(tr.nonterminal), _lib.ptr(tr.ring_state),
                _lib.ptr(tr.running_max), tr.index, src.data_ptr(), _lib.ptr(dev["act"]), _lib.ptr(dev["rew"]),
                _lib.ptr(dev["flag"]), n, _lib.ptr(dev["scratch"]), dev["scratch"].numel(), stream.cuda_stream))
            evt = torch.cuda.Event()
            evt.record(stream)
            stage["evt"][b] = evt
            tr.full = tr.full or tr.index + n >= tr.size
            tr.index = (tr.index + n) % tr.size
        resets = np.flatnonzero(flags)
        self.t = self.t + k if resets.size == 0 else int(k - 1 - resets[-1])

    def _extend_stage(self, chunk, cuda_frames):
        """Pinned staging (two buffers of `chunk` records; frames only for host frames) and the device record buffers."""
        st = getattr(self, "_bulk", None)
        if st is None or st["chunk"] < chunk or (not cuda_frames and st["frames"] is None):
            pin = lambda shape, dt: torch.empty(shape, dtype=dt).pin_memory()   # noqa: E731
            st = dict(chunk=chunk, evt=[None, None],
                      frames=None if cuda_frames else [pin((chunk, FRAME), torch.uint8) for _ in range(2)],
                      act=[pin(chunk, torch.int32) for _ in range(2)], rew=[pin(chunk, torch.float32) for _ in range(2)],
                      flag=[pin(chunk, torch.uint8) for _ in range(2)])
            nbytes = int(self._lib.rb_append_bulk_scratch_bytes(chunk))
            st["dev"] = dict(act=torch.empty(chunk, dtype=torch.int32, device=self.device),
                             rew=torch.empty(chunk, dtype=torch.float32, device=self.device),
                             flag=torch.empty(chunk, dtype=torch.uint8, device=self.device),
                             scratch=torch.empty(nbytes, dtype=torch.uint8, device=self.device))
            old = getattr(self, "_bulk", None)
            if old is not None:   # the old buffers may still feed queued copies
                for e in old["evt"]:
                    if e is not None:
                        e.synchronize()
            self._bulk = st
        return st

    def _check_extend(self, frames, actions, rewards, terminals, final):
        """extend()'s inputs checked and converted: (frames [k, 7056] uint8 tensor, int32, float32 and uint8 flag arrays)."""
        if isinstance(frames, torch.Tensor):
            fr = frames.detach()
            if fr.is_cuda and fr.device != self.device:
                raise ValueError(f"frames are on {fr.device}, the replay on {self.device}")
        else:
            fr = torch.from_numpy(np.ascontiguousarray(frames))
        if fr.is_floating_point():
            raise ValueError("extend takes uint8 frames, already quantised; quantise float frames f in [0, 1] as append "
                             "does: q = (f.astype(np.float32) * np.float32(255)).astype(np.int32).astype(np.uint8)")
        if fr.dtype != torch.uint8:
            raise ValueError(f"frames must be uint8, got {fr.dtype}")
        if not (fr.dim() == 2 and fr.shape[1] == FRAME) and not (fr.dim() == 3 and tuple(fr.shape[1:]) == (84, 84)):
            raise ValueError(f"frames must be [k, 84, 84] or [k, {FRAME}], got {tuple(fr.shape)}")
        k = fr.shape[0]
        fr = fr.reshape(k, FRAME)
        if fr.is_cuda:
            fr = fr.contiguous()

        def host(x, name):
            a = x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)
            if a.shape != (k,):
                raise ValueError(f"{name} must have shape ({k},) like the frames, got {a.shape}")
            return a

        a, r, term = host(actions, "actions"), host(rewards, "rewards"), host(terminals, "terminals")
        if a.dtype.kind not in "iu":
            raise ValueError(f"actions must be integers, got {a.dtype}")
        if k and (a.min() < -2 ** 31 or a.max() >= 2 ** 31):
            raise ValueError("actions must fit int32")
        if r.dtype.kind not in "iuf":
            raise ValueError(f"rewards must be numbers, got {r.dtype}")
        if term.dtype.kind not in "biu":
            raise ValueError(f"terminals must be bool or integers, got {term.dtype}")
        acts = a.astype(np.int32)
        rews = r.astype(np.float64).astype(np.float32)   # float(reward) -> c_float, as append rounds it
        flags = (term != 0).astype(np.uint8)
        if final is not None:
            if not self.bootstrap_truncation:
                raise _lib.RainbowB200Error("extend(final=...) needs args.bootstrap_truncation = True: without it the "
                                            "replay cannot store the final observation a time limit stopped the episode at")
            fin = host(final, "final")
            if fin.dtype.kind not in "biu":
                raise ValueError(f"final must be bool, got {fin.dtype}")
            fin = fin != 0
            idx = np.flatnonzero(fin)
            bad = [(j, why) for j, why in (
                *((j, "is the first record of the call") for j in idx[idx == 0]),
                *((j, "is also terminal") for j in idx[flags[idx] != 0]),
                *((j, "has a nonzero action") for j in idx[acts[idx] != 0]),
                *((j, "has a nonzero reward") for j in idx[rews[idx].view(np.uint32) != 0]),
                *((j, "follows a terminal") for j in idx[(idx > 0) & (flags[idx - 1] != 0)]),
                *((j, "follows another final record") for j in idx[(idx > 0) & fin[idx - 1]]))]
            if bad:
                j, why = min(bad)
                raise ValueError(f"final record {j} {why}: a final observation follows its episode's last transition "
                                 "and carries terminal False, action 0 and reward 0")
            flags[fin] = FINAL
        return fr, acts, rews, flags

    def flush_appends(self):
        """Write the queued transitions (defer_appends=True) with one rb_append_batch launch."""
        if not self._queue:
            return
        q, self._queue = self._queue, []
        self._append_batch(q)
        self._flushed_refs = q   # keep device frames alive until the next flush (the launch is asynchronous)

    def _append_batch(self, q):
        """One rb_append_batch launch (rb_append_batch_trunc with bootstrap_truncation, whose records may be FINAL) for
        the records (frame, action, reward, terminal or FINAL, staging slot or None)."""
        import ctypes as C
        k = len(q)
        tr = self.transitions
        frames = (C.c_void_p * k)(*[e[0].data_ptr() for e in q])   # device or pinned-host pointers (UVA)
        acts = (C.c_int32 * k)(*[e[1] for e in q])
        rews = (C.c_float * k)(*[e[2] for e in q])
        terms = (C.c_int32 * k)(*[int(e[3]) for e in q])
        launch = self._lib.rb_append_batch_trunc if self.bootstrap_truncation else self._lib.rb_append_batch
        _lib.check(launch(
            _lib.ptr(tr.tree), tr.tree_start, tr.size, _lib.ptr(tr.frames), _lib.ptr(tr.timestep), _lib.ptr(tr.action),
            _lib.ptr(tr.reward), _lib.ptr(tr.nonterminal), _lib.ptr(tr.ring_state), _lib.ptr(tr.running_max), frames, acts,
            rews, terms, k, _lib.stream()))
        self._release_stage_slots([e[4] for e in q if e[4] is not None])

    # ---- sample --------------------------------------------------------------------------------
    def _launch_sample(self, ws, u01=None, attempts=0):
        tr = self.transitions
        L = self._lib
        _lib.check(L.rb_tree_sample(
            _lib.ptr(tr.tree), tr.tree_start, tr.size, _lib.ptr(tr.ring_state), self.n, self.history,
            _lib.ptr(u01), attempts, self.seed, _lib.ptr(self._rng_counter), ws.B, float(self.priority_weight),
            _lib.ptr(self._beta_dev), self.max_attempts, _lib.ptr(ws.probs), _lib.ptr(ws.data_idx), _lib.ptr(ws.tree_idx),
            _lib.ptr(ws.weights), _lib.ptr(ws.status), _lib.stream()))

    def _check_shift_pad(self, shift_pad):
        shift_pad = int(shift_pad)
        if not 0 <= shift_pad <= self.MAX_SHIFT_PAD:
            raise ValueError(f"shift_pad must be in [0, {self.MAX_SHIFT_PAD}], got {shift_pad}")
        if shift_pad and self.rng == "numpy":
            raise ValueError("shift_pad > 0 needs rng='philox': the offsets are drawn from the device stream (the reference "
                             "has no augmentation, so there is no numpy stream to reproduce)")
        return shift_pad

    def _check_augmentation(self, shift_pad, intensity, copies):
        """Validated (shift_pad, intensity, (M, K)); ValueError outside the ranges rb_gather_aug takes."""
        shift_pad, intensity = self._check_shift_pad(shift_pad), float(intensity)
        M, K = (int(c) for c in copies)
        if not 0.0 <= intensity <= self.MAX_INTENSITY:   # also refuses NaN
            raise ValueError(f"intensity must be in [0, {self.MAX_INTENSITY}], got {intensity}")
        if not (1 <= M <= self.MAX_AUG_COPIES and 1 <= K <= self.MAX_AUG_COPIES):
            raise ValueError(f"copies (M, K) must each be in [1, {self.MAX_AUG_COPIES}], got {tuple(copies)}")
        if (intensity or (M, K) != (1, 1)) and self.rng == "numpy":
            raise ValueError("intensity > 0 or copies != (1, 1) needs rng='philox': the draws come from the device stream "
                             "(the reference has no augmentation, so there is no numpy stream to reproduce)")
        return shift_pad, intensity, (M, K)

    def _launch_gather(self, ws, shift_pad=0, intensity=0.0, copies=(1, 1), horizon=None):
        """The gather these settings select: rb_gather, rb_gather_shift (shifts only), rb_gather_aug (intensity or
        copies), or with an annealed horizon rb_gather_horizon, which takes every augmentation setting; with
        bootstrap_truncation always rb_gather_trunc, which takes them all too."""
        tr = self.transitions
        shifts, scales = self._aug_buffers(ws, shift_pad, intensity, copies)
        # the n-step window: this replay's n and discount powers (its constant row with bootstrap_truncation), or the
        # horizon's n_max and its current row
        window = (self.n, self.n_step_scaling) if horizon is None else (horizon.n_max, horizon.current)
        if self.bootstrap_truncation and horizon is None:
            window = (self.n, self._fixed_row)
        common = (_lib.ptr(tr.frames), _lib.ptr(tr.timestep), _lib.ptr(tr.action), _lib.ptr(tr.reward),
                  _lib.ptr(tr.nonterminal), tr.size, _lib.ptr(ws.data_idx), ws.B, self.history, window[0],
                  _lib.ptr(window[1]), _lib.ptr(ws.states), _lib.ptr(ws.next_states), _lib.ptr(ws.actions),
                  _lib.ptr(ws.returns), _lib.ptr(ws.nonterminals))
        aug = (shift_pad, intensity, copies[0], copies[1], self.seed, _lib.ptr(self._rng_counter), _lib.ptr(shifts),
               _lib.ptr(scales))
        if self.bootstrap_truncation:
            rc = self._lib.rb_gather_trunc(*common, *aug, _lib.stream())
        elif horizon is not None:
            rc = self._lib.rb_gather_horizon(*common, *aug, _lib.stream())
        elif scales is not None:
            rc = self._lib.rb_gather_aug(*common, *aug, _lib.stream())
        elif shifts is not None:
            rc = self._lib.rb_gather_shift(*common, shift_pad, self.seed, _lib.ptr(self._rng_counter), _lib.ptr(shifts),
                                           _lib.stream())
        else:
            rc = self._lib.rb_gather(*common, _lib.stream())
        _lib.check(rc)

    def _aug_buffers(self, ws, shift_pad, intensity, copies):
        """ws.shifts / ws.scales shaped for the gather these settings select (None where it writes none)."""
        if not shift_pad and not intensity and copies == (1, 1):
            return None, None
        if not intensity and copies == (1, 1):
            if ws.shifts is None or ws.shifts.shape != (2, ws.B, 2):
                ws.shifts = torch.empty((2, ws.B, 2), dtype=torch.int32, device=self.device)
            return ws.shifts, None
        c = max(copies)
        if ws.shifts is None or ws.shifts.shape != (2, c, ws.B, 2):
            ws.shifts = torch.empty((2, c, ws.B, 2), dtype=torch.int32, device=self.device)
        if ws.scales is None or ws.scales.shape != (2, c, ws.B):
            ws.scales = torch.empty((2, c, ws.B), dtype=torch.float32, device=self.device)
        return ws.shifts, ws.scales

    def _check_horizon(self, horizon):
        if horizon is not None and horizon.n_max > self.n:
            raise ValueError(f"the horizon reaches n = {horizon.n_max}, this replay was built for n = {self.n} "
                             "(set args.multi_step_start before building it)")

    def sample_into(self, ws, shift_pad=0, intensity=0.0, copies=(1, 1), horizon=None):
        """Device-RNG sample into caller-owned buffers: two launches, no synchronisation (graph capturable).
        The caller is responsible for push_beta() and flush_appends() (outside any graph capture).
        shift_pad = p > 0 (at most MAX_SHIFT_PAD) augments the states and next states by random shifts (DrQ): each
        observation edge-padded by p pixels and cropped back to 84 x 84 at its own offset drawn on the device
        (rb_gather_shift); `ws.shifts` receives the offsets.  0 gathers exactly as the reference does.
        intensity = s > 0 (at most MAX_INTENSITY) multiplies every observation by 1 + s * clip(N(0, 1), -2, 2) (SPR), and
        copies = (M, K) writes M augmented copies of every state and K of every next state (DrQ's K / M): both go through
        rb_gather_aug, whose draws land in `ws.shifts` and `ws.scales`.  `ws` must have been made for these copies.
        horizon = s (a rainbow_b200.horizon.HorizonSchedule): one step of the annealed horizon.  rb_horizon_advance runs on
        a side branch beside the sampling, and rb_gather_horizon gathers with that step's n and gamma: the returns and next
        states of n_u steps, and the nonterminals in discount form fl32(nonterminal * gamma_u ** n_u), for a loss launched
        with gamma_n = 1.  The sampling itself uses this replay's n (at least s.n_max).  None gathers as before."""
        shift_pad, intensity, copies = self._check_augmentation(shift_pad, intensity, copies)
        if ws.copies != copies:
            raise ValueError(f"the workspace holds copies {ws.copies}, the call asks for {copies}")
        self._check_horizon(horizon)
        if horizon is not None:   # beside rb_tree_sample, which does not read the horizon; joined before the gather
            advanced = _lib.side_branch(horizon.side_stream(), horizon.advance)[1]
        self._launch_sample(ws)
        if horizon is not None:
            torch.cuda.current_stream(self.device).wait_event(advanced)
        self._launch_gather(ws, shift_pad, intensity, copies, horizon)
        self._last = ws
        return ws.as_tuple()

    def sample(self, batch_size, shift_pad=0, intensity=0.0, copies=(1, 1), horizon=None):
        """memory.py:148-155.  Returns (tree_idxs, states, actions, returns, next_states, nonterminals, weights),
        all device tensors (the reference returns tree_idxs as numpy; update_priorities takes either).
        shift_pad, intensity, copies: augmentation as in sample_into(); needs rng="philox" (ValueError otherwise).  With
        copies = (M, K) the states are [M B, ...] and the next states [K B, ...], copy-major.  horizon: as in sample_into()."""
        shift_pad, intensity, copies = self._check_augmentation(shift_pad, intensity, copies)
        self._check_horizon(horizon)
        ws = _SampleWorkspace(int(batch_size), self.history, self.device, copies)
        self.flush_appends()
        self.push_beta()
        if self.rng == "numpy":
            # consume the legacy global generator exactly like np.random.uniform(0, seg, [B]) does
            for _ in range(100000):
                u = torch.from_numpy(np.random.random_sample(ws.B)).to(self.device)
                self._launch_sample(ws, u01=u, attempts=1)
                if int(ws.status[0].item()) == 1:
                    break
            else:  # pragma: no cover
                raise _lib.RainbowB200Error("no valid batch after 100000 draws")
            if horizon is not None:
                horizon.advance()
            self._launch_gather(ws, horizon=horizon)
            self._last = ws
            return ws.as_tuple()
        out = self.sample_into(ws, shift_pad, intensity, copies, horizon)
        if self.strict:
            self.check_last_sample()
        return out

    def sample_gate(self):
        """Device int32 status words of the most recent sample (None in numpy-rng mode, where the host loop only ever
        returns valid batches): element 0 is 0 when that batch was rejected `max_attempts` times.  The kernel has then
        zeroed the batch's importance weights, and handing this tensor as `gate` to update_priorities() / the optimiser
        makes the whole update a no-op -- the device-side stand-in for the reference's unbounded redraw loop
        (memory.py:128-132)."""
        return None if (self._last is None or self.rng == "numpy") else self._last.status

    def rejected_batches(self):
        """Synchronises.  Number of device-RNG batches (since this workspace was created) that stayed invalid after
        `max_attempts` redraws and were therefore skipped."""
        return 0 if self._last is None else int(self._last.status[2].item())

    def check_last_sample(self):
        """Synchronises; raises if the most recent device-RNG sample exhausted max_attempts redraws (strict mode)."""
        if self._last is not None and int(self._last.status[0].item()) != 1:
            raise _lib.RainbowB200Error(
                f"replay sampling rejected {self.max_attempts} consecutive batches (buffer too empty around the "
                "write head, or zero-priority leaves): that batch was skipped (zero weights, no update)")

    # ---- priorities ----------------------------------------------------------------------------
    def update_priorities(self, idxs, priorities, gate=None):
        """memory.py:157-159: raw per-sample losses -> ^omega -> leaves -> propagate to the root.
        `gate` (optional, see sample_gate()): skip the write-back of a rejected batch on the device."""
        if self._queue and not torch.cuda.is_current_stream_capturing():
            self.flush_appends()
        self.transitions.update(idxs, priorities, omega=self.priority_exponent, gate=gate)

    # ---- validation iterator (memory.py:162-180) -------------------------------------------------
    _ITER_CHUNK = 64

    def __iter__(self):
        self.flush_appends()
        self.current_idx = 0
        self._iter_buf = None
        self._iter_base = 0
        return self

    def iter_states(self, first, count):
        """Iterator states (memory.py:166-178) for current_idx = first .. first+count-1 in one launch:
        device float32 [count, history, 84, 84] (backward-only blanking, negative indices wrap)."""
        self.flush_appends()
        tr = self.transitions
        buf = torch.empty((count, self.history, 84, 84), dtype=torch.float32, device=self.device)
        _lib.check(self._lib.rb_iter_states(_lib.ptr(tr.frames), _lib.ptr(tr.timestep), tr.size, int(first), int(count),
                                            self.history, _lib.ptr(buf), _lib.stream()))
        return buf

    def __next__(self):
        if self.current_idx == self.capacity:
            raise StopIteration
        if self._iter_buf is None or self.current_idx >= self._iter_base + self._iter_buf.shape[0]:
            count = min(self._ITER_CHUNK, self.capacity - self.current_idx)
            self._iter_buf, self._iter_base = self.iter_states(self.current_idx, count), self.current_idx
        state = self._iter_buf[self.current_idx - self._iter_base]
        self.current_idx += 1
        return state

    next = __next__

    # ---- pickling (main.py:85-100 pickles the whole object) --------------------------------------
    def __getstate__(self):
        """Own compact layout (plain numpy arrays, structure of arrays).  For a file the REFERENCE can load use
        save_reference_pickle()."""
        self.flush_appends()
        tr = self.transitions
        state = dict(version=1)
        state.update((k, getattr(self, k)) for k in PERSISTENT_HOST)
        state.update(device=str(self.device), rng_counter=int(self._rng_counter.item()), index=tr.index, full=tr.full,
                     max=tr.max)
        state.update((key, getattr(tr, attr).cpu().numpy()) for key, attr in PERSISTENT_ARRAYS)
        if self.bootstrap_truncation:   # absent: off, as in files written before the switch existed
            state["bootstrap_truncation"] = True
        return state

    def _init_runtime(self, rng_counter=0):
        self.n_step_scaling = torch.tensor([self.discount ** i for i in range(self.n)], dtype=torch.float32,
                                           device=self.device)
        if self.bootstrap_truncation:
            self.transitions.final_records = True
        self._fixed_row = self._fixed_horizon_row()
        self.defer_appends, self._queue = False, []
        self._rng_counter = torch.tensor([int(rng_counter)], dtype=torch.int64, device=self.device)
        self._beta_dev = torch.full((1,), float(self.priority_weight), dtype=torch.float32, device=self.device)
        self._beta_pushed = float(self.priority_weight)
        self._lib = _lib.load()
        self._last = None
        self._stage = None

    def __setstate__(self, s):
        if "version" not in s and "transitions" in s:
            return self._setstate_reference(s)
        self.device = _require_cuda(s["device"])
        for k in PERSISTENT_HOST:
            setattr(self, k, s[k])
        self.bootstrap_truncation = bool(s.get("bootstrap_truncation", False))
        self.transitions = SegmentTree(self.capacity, self.device)
        self.transitions.load_arrays(**{key: s[key] for key, _ in PERSISTENT_ARRAYS}, index=s["index"], full=s["full"],
                                     t_episode=s["t"], max_value=s["max"])
        self._init_runtime(s["rng_counter"])

    def _setstate_reference(self, s):
        """A memory file written by the REFERENCE (its ReplayMemory.__dict__, memory.py:93-102, with the AoS
        Transition_dtype `data` and the truncated `sum_tree` of memory.py:13-20): rebuilt in HBM.  A CPU device in the
        file is mapped to the current CUDA device (the replay has no host variant)."""
        dev = torch.device(s.get("device", "cuda"))
        self.device = _require_cuda(dev if dev.type == "cuda" else "cuda")
        self.capacity, self.history, self.discount, self.n = int(s["capacity"]), int(s["history"]), s["discount"], int(s["n"])
        self.priority_weight, self.priority_exponent, self.t = s["priority_weight"], s["priority_exponent"], int(s["t"])
        self.rng, self.max_attempts, self.strict = "philox", 64, False
        self.bootstrap_truncation = False
        self.seed = int(torch.initial_seed()) & (2 ** 64 - 1)
        tr = s["transitions"]
        if isinstance(tr, SegmentTree):
            tr._materialise(self.device, self.t)
        else:   # any object carrying the reference's fields
            fields = {k: getattr(tr, k) for k in ("index", "size", "full", "sum_tree", "data", "max")}
            tr = SegmentTree(int(fields["size"]), self.device)
            tr.load_arrays(**reference_fields_to_ring(fields, t=self.t))
        self.transitions = tr
        self._init_runtime()

    def reference_state(self, device="cpu"):
        """(ReplayMemory.__dict__, SegmentTree.__dict__) exactly as the reference's objects hold them.  Refuses a ring
        holding final-observation records (append_truncated): the reference's memory has no way to represent them."""
        if self.holds_final_records():
            raise _lib.RainbowB200Error("the replay holds final-observation records (append_truncated), which the "
                                        "reference's memory cannot represent: no reference-format copy of it can be made")
        dev = torch.device(device)
        mem = dict(device=dev, capacity=self.capacity, history=self.history, discount=self.discount, n=self.n,
                   priority_weight=self.priority_weight, priority_exponent=self.priority_exponent, t=self.t,
                   n_step_scaling=self.n_step_scaling.to(dev))
        return mem, self.transitions.__getstate__()


def save_reference_pickle(mem, file, device="cpu", protocol=None):
    """Write `mem` as a pickle the UNMODIFIED reference loads with pickle.load (main.py:85-91): the stream names the
    classes `memory.ReplayMemory` / `memory.SegmentTree` and carries the reference's own field layout, so inside the
    reference process it unpickles into the reference's classes (and, with dropin/ on the path, into ours)."""
    import pickle
    import sys
    import types
    mem_state, tree_state = mem.reference_state(device)
    stand_in = types.ModuleType("memory")
    tree_cls = type("SegmentTree", (), {"__module__": "memory"})
    mem_cls = type("ReplayMemory", (), {"__module__": "memory"})
    stand_in.SegmentTree, stand_in.ReplayMemory = tree_cls, mem_cls
    tree = tree_cls()
    tree.__dict__.update(tree_state)
    obj = mem_cls()
    obj.__dict__.update(mem_state, transitions=tree)
    saved = sys.modules.get("memory")
    sys.modules["memory"] = stand_in      # pickle verifies that memory.ReplayMemory is the class being written
    try:
        pickle.dump(obj, file, protocol=protocol)
    finally:
        if saved is None:
            del sys.modules["memory"]
        else:
            sys.modules["memory"] = saved


def ring_to_reference_fields(state):
    """Host-side helper for format exchange: the pickled dict above -> the fields of the reference's
    SegmentTree (memory.py:13-20): index, size, full, tree_start, sum_tree, data (AoS Transition_dtype), max."""
    size = state["capacity"]
    data = np.zeros(size, dtype=Transition_dtype)
    data["timestep"] = state["timestep"]
    data["state"] = np.asarray(state["frames"]).reshape(size, 84, 84)
    data["action"] = state["action"]
    data["reward"] = state["reward"]
    data["nonterminal"] = np.asarray(state["nonterminal"]).astype(np.bool_)
    return dict(index=state["index"], size=size, full=state["full"], tree_start=2 ** (size - 1).bit_length() - 1,
                sum_tree=np.asarray(state["sum_tree"], dtype=np.float32), data=data, max=state["max"])


def reference_fields_to_ring(fields, t=0):
    """Inverse of ring_to_reference_fields: SegmentTree attributes of the reference -> load_arrays kwargs."""
    data = fields["data"]
    size = int(fields["size"])
    return dict(sum_tree=fields["sum_tree"], frames=np.ascontiguousarray(data["state"]).reshape(size, FRAME),
                timestep=data["timestep"], action=data["action"], reward=data["reward"],
                nonterminal=data["nonterminal"].astype(np.uint8), index=fields["index"], full=fields["full"],
                t_episode=t, max_value=fields["max"])
