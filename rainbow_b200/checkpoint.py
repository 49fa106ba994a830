"""Exact-resume checkpoints of the learner and its replay (Agent.save_checkpoint / Agent.load_checkpoint).

A checkpoint holds everything that decides the next update's result and nothing else (DESIGN.md §9): the online
parameters (the whole flat buffer, padding included), the target net's parameters, the Adam moments and step count, both
nets' noise streams (seed, Philox counter, factor vectors, epsilon buffers) and the online net's pending-draw flag, the
parameter-reset key and count, the learn-statistics ring, and -- when a ReplayMemory is passed -- the replay's device arrays, ring state, sampling stream and host mirrors.

Layout: `path/rank{r}/` per data-parallel rank, holding `manifest.json` (format version, world size, rank, optimiser layout,
structural config, host scalars, a save id shared by all ranks of one save, per array its dtype, shape and SHA-256, and a
digest of the manifest itself) and one `.npy` file per array, named after the array.  There is no pickle anywhere: the
files are plain `.npy` (np.load(allow_pickle=False) reads them), their headers are parsed by numpy's own `.npy` reader and
object arrays are refused, so loading somebody else's checkpoint cannot run code.

Writes go to a temporary sibling directory that is renamed into place once every file is complete: a save interrupted by
preemption leaves the previous checkpoint intact and never a partial one that looks valid.  Every byte moves between the
device and the file through one bounded (pinned) staging buffer, in chunks, both ways: a 1M-transition replay (7.07 GB) needs
CHUNK_BYTES of extra host memory per rank, not 7 GB.

Loading opens the rank directory once and validates everything (manifest digest, structure, every host scalar, every
file's header and checksum) before its first device write, then restores from the same open files; a refusal raises
RainbowB200Error and leaves every device and host field as it was.  Under data parallelism the ranks agree with one MIN
all-reduce of the ok flag and the save id: either all restore the same save or all raise.
"""
import hashlib
import json
import math
import os
import shutil
import uuid

import numpy as np
import torch

from . import _lib
from .memory import PERSISTENT_ARRAYS, PERSISTENT_HOST, PERSISTENT_ROLES

FORMAT = "rainbow_b200.checkpoint"
VERSION = 1
MANIFEST = "manifest.json"
CHUNK_BYTES = 64 << 20

_Error = _lib.RainbowB200Error


# ---- host part: arrays, manifest, directories (no GPU needed) ------------------------------------------------------------
class Staging:
    """The one bounded host buffer every array moves through, in chunks of `chunk_bytes` (page-locked when CUDA is
    available, so device copies run at full PCIe speed)."""

    def __init__(self, chunk_bytes=CHUNK_BYTES, pin=None):
        pin = torch.cuda.is_available() if pin is None else pin
        self.buf = torch.empty(max(1, int(chunk_bytes)), dtype=torch.uint8, pin_memory=pin)
        self.chunk = self.buf.numel()
        self.mv = memoryview(self.buf.numpy())


def _np_dtype(torch_dtype):
    return torch.empty(0, dtype=torch_dtype).numpy().dtype


def _as_tensor(src):
    if isinstance(src, np.ndarray):
        if src.dtype.hasobject:
            raise _Error(f"refusing to checkpoint an object array ({src.dtype}): only plain numeric arrays are stored")
        return torch.from_numpy(np.ascontiguousarray(src))
    if not isinstance(src, torch.Tensor):
        raise _Error(f"cannot checkpoint a {type(src).__name__}: arrays must be tensors or numeric numpy arrays")
    return src


def _byte_view(t):
    if not t.is_contiguous():
        raise _Error("checkpointed tensors must be contiguous")
    if t.numel() == 0:
        return torch.empty(0, dtype=torch.uint8, device=t.device)
    return t.reshape(-1).view(torch.uint8)


def write_array(path, src, staging):
    """Write a tensor (any device) or numeric numpy array to a new `.npy` file through `staging`; returns its manifest
    entry {dtype, shape, sha256} (the checksum covers the data bytes)."""
    t = _as_tensor(src)
    dt = _np_dtype(t.dtype)
    flat = _byte_view(t)
    h = hashlib.sha256()
    with open(path, "xb") as f:
        np.lib.format.write_array_header_1_0(f, dict(descr=np.lib.format.dtype_to_descr(dt), fortran_order=False,
                                                     shape=tuple(t.shape)))
        n = flat.numel()
        for off in range(0, n, staging.chunk):
            k = min(staging.chunk, n - off)
            staging.buf[:k].copy_(flat[off:off + k])     # synchronous: the buffer is reused by the next chunk
            h.update(staging.mv[:k])
            f.write(staging.mv[:k])
        f.flush()
        os.fsync(f.fileno())
    return dict(dtype=dt.str, shape=list(t.shape), sha256=h.hexdigest())


def _read_header(f, name):
    """dtype, shape, data offset and data size of an open `.npy` file.  The header is parsed by numpy's own reader
    (np.lib.format, the parser behind np.load; nothing is ever unpickled); object and Fortran-ordered arrays are refused,
    and the file must hold exactly the bytes the header describes."""
    f.seek(0)
    try:
        version = np.lib.format.read_magic(f)
        if version == (1, 0):
            shape, fortran, dtype = np.lib.format.read_array_header_1_0(f)
        elif version == (2, 0):
            shape, fortran, dtype = np.lib.format.read_array_header_2_0(f)
        else:
            raise ValueError(f".npy format version {version} is not part of the checkpoint format")
    except (OSError, ValueError, EOFError, SyntaxError) as e:
        raise _Error(f"{name}: not a readable .npy array ({e})") from e
    if dtype.hasobject or (fortran and len(shape) > 1):
        raise _Error(f"{name}: object or Fortran-ordered arrays are not part of the format")
    offset = f.tell()
    nbytes = int(np.prod(shape, dtype=np.int64)) * dtype.itemsize
    size = os.fstat(f.fileno()).st_size
    if size != offset + nbytes:
        raise _Error(f"{name}: {size} bytes on disk, the header describes {offset + nbytes} (truncated or padded)")
    return dtype, tuple(shape), offset, nbytes


def _stream(f, name, offset, nbytes, staging, sink=None, hashing=True):
    h = hashlib.sha256() if hashing else None
    f.seek(offset)
    done = 0
    while done < nbytes:
        k = min(staging.chunk, nbytes - done)
        if f.readinto(staging.mv[:k]) != k:
            raise _Error(f"{name}: truncated")
        if h is not None:
            h.update(staging.mv[:k])
        if sink is not None:
            sink(done, k)
        done += k
    return None if h is None else h.hexdigest()


def _check_header(f, name, entry):
    dtype, shape, offset, nbytes = _read_header(f, name)
    if dtype.str != entry["dtype"] or list(shape) != list(entry["shape"]):
        raise _Error(f"{name}: holds {dtype.str} {list(shape)}, the manifest says {entry['dtype']} {entry['shape']}")
    return offset, nbytes


def verify_array(f, entry, staging, name="array"):
    """Header of the open file `f` against the manifest entry, then the SHA-256 of its data bytes (read through
    `staging`, nothing else written)."""
    offset, nbytes = _check_header(f, name, entry)
    if _stream(f, name, offset, nbytes, staging) != entry["sha256"]:
        raise _Error(f"{name}: SHA-256 mismatch (the file is corrupt)")


def read_array_into(f, entry, dst, staging, name="array"):
    """Copy the data of the open, already verified `.npy` file `f` into `dst` in place (chunked through `staging`)."""
    offset, nbytes = _check_header(f, name, entry)
    flat = _byte_view(dst)
    if flat.numel() != nbytes:
        raise _Error(f"{name}: {nbytes} bytes for a {flat.numel()}-byte destination")
    _stream(f, name, offset, nbytes, staging, hashing=False,
            sink=lambda off, k: flat[off:off + k].copy_(staging.buf[:k]))    # synchronous, as in write_array


def _digest(man):
    """SHA-256 of the manifest body (every key but the digest itself, canonical JSON)."""
    body = {k: v for k, v in man.items() if k != "digest"}
    return hashlib.sha256(json.dumps(body, sort_keys=True, separators=(",", ":")).encode()).hexdigest()


def _parse_manifest(raw, directory):
    try:
        man = json.loads(raw)
    except ValueError as e:
        raise _Error(f"no readable checkpoint manifest in {directory} ({e})") from e
    if not isinstance(man, dict) or man.get("format") != FORMAT:
        raise _Error(f"{directory}: not a {FORMAT} manifest")
    if man.get("version") != VERSION:
        raise _Error(f"{directory}: checkpoint format version {man.get('version')}, this build reads version {VERSION}")
    if man.get("digest") != _digest(man):
        raise _Error(f"{directory}: manifest digest mismatch (the manifest is corrupt or was edited)")
    if not isinstance(man.get("arrays"), dict):
        raise _Error(f"{directory}: manifest without an array table")
    return man


class CheckpointDir:
    """One rank directory, opened once.  The manifest and every array file are opened through one directory descriptor
    and stay open until close(): the verifying read and the restoring read go to the same files, so a save that renames a
    newer directory into place meanwhile cannot leak into this load."""

    def __init__(self, directory):
        self.directory = directory
        self._files = {}
        try:
            self._dfd = os.open(directory, os.O_RDONLY | os.O_DIRECTORY)
        except OSError as e:
            raise _Error(f"no checkpoint directory {directory} ({e})") from e
        try:
            with self._open(MANIFEST) as f:
                self.manifest = _parse_manifest(f.read(), directory)
        except BaseException:
            self.close()
            raise

    def _open(self, fname):
        try:
            return os.fdopen(os.open(fname, os.O_RDONLY, dir_fd=self._dfd), "rb")
        except FileNotFoundError as e:
            raise _Error(f"{fname} is missing from {self.directory}") from e
        except OSError as e:
            raise _Error(f"{fname} in {self.directory} cannot be opened ({e})") from e

    def _file(self, name):
        if name not in self._files:
            fname = self.manifest["arrays"][name].get("file")
            if fname != name + ".npy":      # the naming rule: no other path is ever opened
                raise _Error(f"array '{name}': file {fname!r} breaks the format's naming rule ('{name}.npy')")
            self._files[name] = self._open(fname)
        return self._files[name]

    def verify(self, expected, staging):
        """Every array of `expected` {name: (dtype str, shape)} must be in the manifest with that dtype and shape, and its
        file must match the manifest entry's header and checksum.  Reads only."""
        arrays = self.manifest["arrays"]
        for name, (dtype, shape) in expected.items():
            e = arrays.get(name)
            if not isinstance(e, dict):
                raise _Error(f"array '{name}' is missing from the checkpoint")
            if e.get("dtype") != dtype or list(e.get("shape", ())) != list(shape):
                raise _Error(f"array '{name}': checkpoint has {e.get('dtype')} {e.get('shape')}, this object needs "
                             f"{dtype} {list(shape)}")
            verify_array(self._file(name), e, staging, name + ".npy")

    def read_into(self, name, dst, staging):
        read_array_into(self._file(name), self.manifest["arrays"][name], dst, staging, name + ".npy")

    def close(self):
        for f in self._files.values():
            f.close()
        self._files = {}
        if getattr(self, "_dfd", None) is not None:
            os.close(self._dfd)
            self._dfd = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def read_manifest(directory):
    with CheckpointDir(directory) as d:
        return d.manifest


def _fsync_dir(directory):
    fd = os.open(directory, os.O_RDONLY)
    try:
        os.fsync(fd)
    finally:
        os.close(fd)


def write_dir(final, arrays, meta, chunk_bytes=CHUNK_BYTES):
    """Write {name: tensor / array} and the manifest `meta` into a temporary sibling of `final` and rename it into place.
    An existing `final` is replaced only after the new directory is complete: it is renamed to a `.{name}.old-*` sibling,
    the new one takes its place, and the old one is deleted.  A process killed between those two renames leaves only the
    `.old-*` directory, complete, which rank_directory() falls back to.  On any failure the temporary directory is removed
    and `final` is left as it was."""
    parent = os.path.dirname(os.path.abspath(final))
    tmp = os.path.join(parent, f".{os.path.basename(final)}.partial-{os.getpid()}-{uuid.uuid4().hex[:8]}")
    os.mkdir(tmp)
    try:
        staging = Staging(chunk_bytes)
        table = {}
        for name, src in arrays.items():
            entry = write_array(os.path.join(tmp, name + ".npy"), src, staging)
            table[name] = dict(file=name + ".npy", **entry)
        man = dict(meta, format=FORMAT, version=VERSION, arrays=table)
        man["digest"] = _digest(man)
        with open(os.path.join(tmp, MANIFEST), "x") as f:
            json.dump(man, f, indent=1, sort_keys=True)
            f.flush()
            os.fsync(f.fileno())
        _fsync_dir(tmp)
        if os.path.exists(final):
            old = os.path.join(parent, f".{os.path.basename(final)}.old-{uuid.uuid4().hex[:8]}")
            os.rename(final, old)
            os.rename(tmp, final)
            shutil.rmtree(old, ignore_errors=True)
        else:
            os.rename(tmp, final)
        _fsync_dir(parent)
    except BaseException:
        shutil.rmtree(tmp, ignore_errors=True)
        raise


# ---- the learner and the replay ------------------------------------------------------------------------------------------
def _learner_arrays(agent):
    """The learner's device state as the live tensors (the checkpoint writes them and restores into them in place)."""
    on, tg, opt = agent.online_net, agent.target_net, agent.optimiser
    sd = opt.state_dict(clone=False)
    arrays = {"online.flat_param": opt.flat_param}          # every online parameter is a view into it (+ zero padding)
    arrays.update((f"target.{n}", p.data) for n, p in tg.named_parameters())
    arrays["optimiser.exp_avg"], arrays["optimiser.exp_avg_sq"] = sd["exp_avg"], sd["exp_avg_sq"]
    for tag, net in (("online", on), ("target", tg)):
        arrays[f"{tag}.noise_counter"] = net._noise_counter
        arrays[f"{tag}.f_in"], arrays[f"{tag}.f_out"] = net._f_in, net._f_out
        # weight_epsilon / bias_epsilon as they are (outer products of the factors unless marked stale, or what
        # load_state_dict put there): the library head reads them as the next update's noise
        arrays.update((f"{tag}.{n}", b) for n, b in net.named_buffers() if n.endswith("_epsilon"))
    if agent._stats is not None:
        arrays["learn_stats.ring"] = agent._stats["buf"]    # record 0 holds the device counter
    # not saved: flat_grad (every update overwrites it), the clip + Adam partials, learn-stats scratch and head tickets
    # (zero between launches), and the peer optimiser's epoch and flag words -- synchronisation state shared with the other
    # ranks' kernels: writing them in place would deadlock or corrupt rb_peer_adam_gather
    return arrays


def _replay_arrays(mem):
    tr = mem.transitions
    arrays = {f"replay.{key}": getattr(tr, attr) for key, attr in PERSISTENT_ARRAYS}
    arrays["replay.ring_state"] = tr.ring_state[:4]      # head, full, t_episode, appended; [4] is a launch ticket (zero)
    arrays["replay.running_max"] = tr.running_max
    arrays["replay.rng_counter"] = mem._rng_counter
    return arrays


def _structure(agent, mem):
    on = agent.online_net
    s = dict(architecture=on.architecture, hidden_size=on.hidden_size, atoms=agent.atoms, actions=agent.action_space,
             history_length=agent.history, flat_numel=agent.optimiser.numel)
    if mem is not None:
        s["replay"] = {k: getattr(mem, k) for k, role in PERSISTENT_ROLES if role == "structure"}
    return s


def _meta(agent, mem):
    on, opt = agent.online_net, agent.optimiser
    sd = opt.state_dict(clone=False)
    st = agent._stats
    learner = dict(learn_calls=agent._learn_calls, online_noise_seed=on.noise_seed,
                   target_noise_seed=agent.target_net.noise_seed, online_noise_pending=bool(on._noise_pending),
                   online_eps_stale=bool(on._eps_stale), target_eps_stale=bool(agent.target_net._eps_stale),
                   optimiser_step=sd["step"], learn_stats_capacity=agent.learn_stats_capacity,
                   learn_stats_read=0 if st is None else st["read"])
    hyper = dict(learning_rate=opt.lr, adam_eps=opt.eps, betas=list(opt.betas), norm_clip=agent.norm_clip,
                 discount=agent.discount, multi_step=agent.n, batch_size=agent.batch_size, V_min=agent.Vmin,
                 V_max=agent.Vmax)
    if agent.augment_shift:   # only when on: manifests of runs without augmentation stay as they were
        hyper["augment_shift"] = agent.augment_shift
    if agent.augment_intensity:
        hyper["augment_intensity"] = agent.augment_intensity
    if agent.augment_copies != (1, 1):
        hyper["augment_m"], hyper["augment_k"] = agent.augment_copies
    if agent.target_tau:
        hyper["target_tau"] = agent.target_tau
    if agent.reset_interval:
        hyper["reset_interval"] = agent.reset_interval
    if agent.reset_shrink[0] != 1.0:
        hyper["reset_shrink_encoder"] = agent.reset_shrink[0]
    if agent.reset_shrink[1] != 0.0:
        hyper["reset_shrink_head"] = agent.reset_shrink[1]
    if agent.weight_decay:
        hyper["weight_decay"] = agent.weight_decay
    if agent.reset_optimizer:
        hyper["reset_optimizer"] = True
    if agent.redo_interval:
        hyper["redo_interval"] = agent.redo_interval
    if agent.redo_tau != 0.1:
        hyper["redo_tau"] = agent.redo_tau
    if agent.quantile:   # absent: categorical
        hyper["distribution"], hyper["quantile_kappa"] = agent.distribution, agent.quantile_kappa
    if agent.value_transform is not None:   # absent: no value rescaling
        hyper["value_transform"], hyper["value_transform_eps"] = agent.value_transform, agent.value_transform_eps
    if agent.quantile_average_copies:   # absent: the quantile loss does not average copies
        hyper["quantile_average_copies"] = True
    if agent.munchausen is not None:   # absent: no Munchausen targets
        hyper["munchausen_alpha"], hyper["munchausen_temperature"], hyper["munchausen_clip"] = agent.munchausen
    if agent.risk is not None:   # absent: the mean selects (no risk measure)
        hyper["risk_measure"], hyper["risk_eta"] = agent.risk
    hlg = getattr(agent, "hl_gauss_sigma", None)   # an agent without the attribute reads as off
    if hlg is not None:   # absent: C51's projection
        hyper["categorical_target"], hyper["hl_gauss_sigma"] = "hl_gauss", hlg
    if getattr(agent, "two_hot", False):   # two-hot targets record the switch alone
        hyper["categorical_target"] = "two_hot"
    if getattr(agent, "cql_alpha", None) is not None:   # absent: CQL's regulariser off
        hyper["cql_alpha"] = agent.cql_alpha
    if agent.bootstrap_truncation:   # absent: off
        hyper["bootstrap_truncation"] = True
    if agent.redo_interval or agent.redo_count:   # the index of the next recycling pass: the counter of its draws
        learner["redo_count"] = agent.redo_count
    if opt.grouped:   # the group optimiser's bias-correction counts, [encoder, head]
        learner["optimiser_group_steps"] = opt.group_step_counts()
    hz = agent._horizon
    if hz is not None:   # the annealed horizon's options (when not their defaults) and the cycle step of the next update
        hyper["anneal_steps"] = hz.T
        if hz.n0 != hz.n1:
            hyper["multi_step_start"] = hz.n0
        if hz.g0 != hz.g1:
            hyper["discount_start"] = hz.g0
        learner["horizon_step"] = hz.step
    # always: the key comes from the caller's torch seed, and a resumed process may have another one.  Manifests written
    # before these keys existed have neither, which load() reads as no reset yet, with the live seed.
    learner.update(reset_seed=agent.reset_seed, reset_count=agent.reset_count)
    meta = dict(world_size=agent.sync.world_size, rank=agent.sync.rank, optimiser=sd["layout"],
                structure=_structure(agent, mem), hyper_parameters=hyper, learner=learner, replay=None)
    if mem is not None:
        tr = mem.transitions
        replay = {k: getattr(mem, k) for k in PERSISTENT_HOST}
        replay.update(index=tr.index, full=tr.full)
        if mem.bootstrap_truncation:   # absent: off, and then the ring holds no final-observation record
            replay["bootstrap_truncation"] = True
            replay["final_records"] = mem.holds_final_records()
        meta["replay"] = replay
    return meta


def _save_id(agent):
    """One id for all ranks' directories of one save: rank 0 draws it, the others receive it.  load() refuses rank
    directories whose ids differ -- say, rank 0 renamed into place at update N + 1 and rank 1 still at update N after a
    preemption between the ranks' renames -- instead of restoring diverged replicas."""
    sid = torch.tensor([int.from_bytes(os.urandom(8), "little") >> 2 | 1], dtype=torch.int64, device=agent.device)
    if agent.sync.enabled:
        torch.distributed.broadcast(sid, src=0, group=agent.sync.group)
    return int(sid.item())


def save(agent, path, mem=None, chunk_bytes=CHUNK_BYTES):
    """Agent.save_checkpoint: `path/rank{r}/`, written atomically.  Under data parallelism every rank calls it."""
    if mem is not None:
        mem.flush_appends()   # queued appends belong to the replay's state
    sid = _save_id(agent)
    torch.cuda.synchronize(agent.device)
    arrays = _learner_arrays(agent)
    if mem is not None:
        arrays.update(_replay_arrays(mem))
    meta = dict(_meta(agent, mem), save_id=sid)
    created = not os.path.isdir(path)
    os.makedirs(path, exist_ok=True)
    try:
        write_dir(os.path.join(path, f"rank{agent.sync.rank}"), arrays, meta, chunk_bytes)
    except BaseException:
        if created:
            try:
                os.rmdir(path)     # only if empty: another rank's complete directory stays
            except OSError:
                pass
        raise


def rank_directory(path, rank):
    """`path/rank{rank}`, or -- when a process was killed between the two renames that replace it (write_dir) -- the
    complete previous directory left under its `.rank{rank}.old-*` name."""
    final = os.path.join(path, f"rank{rank}")
    if os.path.isdir(final) or not os.path.isdir(path):
        return final
    prefix = f".rank{rank}.old-"
    old = [os.path.join(path, n) for n in os.listdir(path) if n.startswith(prefix)]
    return max(old, key=os.path.getmtime) if old else final


def _spec(t):
    return _np_dtype(t.dtype).str, list(t.shape)


def _is_int(v, lo, hi):
    return isinstance(v, int) and not isinstance(v, bool) and lo <= v < hi


_U63, _U64 = 2 ** 63, 2 ** 64
# every host scalar a restore applies: (section, key) -> check
_SCALARS = {
    ("learner", "learn_calls"): lambda v, m: _is_int(v, 0, _U63),
    ("learner", "online_noise_seed"): lambda v, m: _is_int(v, 0, _U63),
    ("learner", "target_noise_seed"): lambda v, m: _is_int(v, 0, _U63),
    ("learner", "online_noise_pending"): lambda v, m: isinstance(v, bool),
    ("learner", "online_eps_stale"): lambda v, m: isinstance(v, bool),
    ("learner", "target_eps_stale"): lambda v, m: isinstance(v, bool),
    ("learner", "optimiser_step"): lambda v, m: _is_int(v, 0, _U63),
    ("learner", "learn_stats_capacity"): lambda v, m: _is_int(v, 0, 2 ** 31),
    ("learner", "learn_stats_read"): lambda v, m: _is_int(v, 0, _U63),
    ("learner", "reset_seed"): lambda v, m: v is None or _is_int(v, 0, _U63),      # absent (both): an older manifest
    ("learner", "reset_count"): lambda v, m: v is None or _is_int(v, 0, _U63),
    ("learner", "horizon_step"): lambda v, m: v is None or _is_int(v, 0, _U63),     # absent: annealing off, or step 0
    ("learner", "redo_count"): lambda v, m: v is None or _is_int(v, 0, _U63),       # absent: no recycling pass yet
    ("replay", "t"): lambda v, m: _is_int(v, 0, _U63),
    ("replay", "seed"): lambda v, m: _is_int(v, 0, _U64),
    ("replay", "priority_weight"): lambda v, m: isinstance(v, (int, float)) and not isinstance(v, bool) and math.isfinite(v),
    ("replay", "index"): lambda v, m: _is_int(v, 0, m.capacity),
    ("replay", "full"): lambda v, m: isinstance(v, bool),
}
# a replay field that gets the "state" role in memory.PERSISTENT_ROLES must get its check here
assert {("replay", k) for k, role in PERSISTENT_ROLES if role == "state"} <= set(_SCALARS)


def check_reset_scalars(learner):
    """The reset key and count come as a pair: both (this format) or neither (a manifest written before they existed).  A
    count without its key would resume the reset schedule with the live key, a key without a count with index 0."""
    if (learner.get("reset_seed") is None) != (learner.get("reset_count") is None):
        raise _Error("manifest learner.reset_seed and learner.reset_count must be given together (or both be absent)")


def check_group_steps(learner):
    """learner.optimiser_group_steps, when present: [encoder, head], two ints in [0, optimiser_step] (a group's count
    restarts at a reset and never passes the applied steps).  Absent: a manifest of a run without the group optimiser,
    which loads with both counts equal to optimiser_step."""
    v = learner.get("optimiser_group_steps")
    if v is None:
        return
    step = learner.get("optimiser_step")
    if not (isinstance(v, list) and len(v) == 2 and _is_int(step, 0, _U63) and all(_is_int(c, 0, step + 1) for c in v)):
        raise _Error(f"manifest learner.optimiser_group_steps = {v!r} must be two ints in [0, optimiser_step = {step!r}]")


def _validate(agent, mem, man):
    """Every check of load(), none of which writes anything; returns the expected {array name: (dtype, shape)}."""
    world, rank = agent.sync.world_size, agent.sync.rank
    if man.get("world_size") != world or man.get("rank") != rank:
        raise _Error(f"checkpoint of rank {man.get('rank')} of {man.get('world_size')}, this learner is rank {rank} of "
                     f"{world} (resharding is not supported)")
    if not _is_int(man.get("save_id"), 1, _U63):
        raise _Error("manifest without a valid save_id")
    want, have = _structure(agent, mem), dict(man.get("structure") or {})
    if mem is not None and (have.get("replay") is None or not isinstance(man.get("replay"), dict)):
        raise _Error("the checkpoint holds no replay memory")
    for key in want:
        if have.get(key) != want[key]:
            raise _Error(f"{key} differs: checkpoint {have.get(key)}, live {want[key]}")
    # the parameter shapes are the same under both losses: without this a C51 net would load as quantiles, or back
    dist = (man.get("hyper_parameters") or {}).get("distribution", "categorical")
    if dist != agent.distribution:
        raise _Error(f"distribution differs: checkpoint {dist!r}, live {agent.distribution!r}")
    # likewise a net trained in h units (value rescaling) would load silently as a plain one, or under another eps
    hyper = man.get("hyper_parameters") or {}
    vt = (hyper.get("value_transform"), hyper.get("value_transform_eps"))
    if vt != (agent.value_transform, agent.value_transform_eps):
        raise _Error(f"value transform differs: checkpoint {vt}, live {(agent.value_transform, agent.value_transform_eps)}")
    # and a net trained against the quantile-wise average of K target copies would resume under another loss
    qavg = hyper.get("quantile_average_copies", False)
    if qavg is not agent.quantile_average_copies:
        raise _Error(f"quantile_average_copies differs: checkpoint {qavg!r}, live {agent.quantile_average_copies!r}")
    # and one trained against Munchausen targets, or under other (alpha, temperature, clip)
    munch = tuple(hyper.get(k) for k in ("munchausen_alpha", "munchausen_temperature", "munchausen_clip"))
    live = agent.munchausen or (None, None, None)
    if munch != live:
        raise _Error(f"munchausen (alpha, temperature, clip) differs: checkpoint {munch}, live {live}")
    # and one whose policy read its distribution through another risk measure, or through none
    risk = (hyper.get("risk_measure"), hyper.get("risk_eta"))
    live = agent.risk or (None, None)
    if risk != live:
        raise _Error(f"risk measure (measure, eta) differs: checkpoint {risk}, live {live}")
    # and one trained against another categorical target, or with another HL-Gauss width
    hlg = (hyper.get("categorical_target"), hyper.get("hl_gauss_sigma"))
    live = getattr(agent, "hl_gauss_sigma", None)
    live = (None, None) if live is None else ("hl_gauss", live)
    if getattr(agent, "two_hot", False):
        live = ("two_hot", None)
    if hlg != live:
        raise _Error(f"categorical target (categorical_target, hl_gauss_sigma) differs: checkpoint {hlg}, live {live}")
    if hyper.get("cql_alpha") != getattr(agent, "cql_alpha", None):
        raise _Error(f"cql_alpha differs: checkpoint {hyper.get('cql_alpha')}, live {getattr(agent, 'cql_alpha', None)}")
    # a ring with final-observation records means nothing to a replay that gathers without cutting windows at them
    if mem is not None and (man.get("replay") or {}).get("final_records") and not mem.bootstrap_truncation:
        raise _Error("the checkpoint's replay holds final-observation records (args.bootstrap_truncation) and this "
                     "replay was built without args.bootstrap_truncation")
    layout = agent.optimiser.state_dict(clone=False)["layout"]
    if man.get("optimiser") != layout:
        raise _Error(f"optimiser layout differs: checkpoint {man.get('optimiser')}, this learner {layout}")
    for (section, key), ok in _SCALARS.items():
        if section == "replay" and mem is None:
            continue
        v = (man.get(section) or {}).get(key)
        if not ok(v, mem):
            raise _Error(f"manifest {section}.{key} = {v!r} is missing or out of range")
    check_reset_scalars(man["learner"])
    check_group_steps(man["learner"])
    cap = man["learner"]["learn_stats_capacity"]
    expected = {n: _spec(t) for n, t in _learner_arrays(agent).items() if n != "learn_stats.ring"}
    if cap:
        expected["learn_stats.ring"] = ("<i4", [(cap + 1) * _lib.LEARN_STATS_RECORD_BYTES // 4])
    if mem is not None:
        expected.update((n, _spec(t)) for n, t in _replay_arrays(mem).items())
    extra = {n for n in man["arrays"] if n not in expected and not (mem is None and n.startswith("replay."))}
    if extra:
        raise _Error(f"unexpected arrays in the checkpoint: {sorted(extra)}")
    return expected


def _agree(agent, err, sid):
    """Under data parallelism: one MIN all-reduce of [ok, save id, -save id].  Every rank raises unless all validated
    and all hold directories of the same save."""
    if not agent.sync.enabled:
        return err
    ok = err is None
    t = torch.tensor([int(ok), sid if ok else 0, -sid if ok else 0], dtype=torch.int64, device=agent.device)
    torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MIN, group=agent.sync.group)
    all_ok, lo, hi = int(t[0]), int(t[1]), -int(t[2])
    if ok and not all_ok:
        return _Error("refused on another rank")
    if ok and lo != hi:
        return _Error("the rank directories come from different saves (a save was interrupted between the ranks' "
                      "renames); load an earlier checkpoint")
    return err


def load(agent, path, mem=None, chunk_bytes=CHUNK_BYTES):
    """Agent.load_checkpoint: validate everything, agree across ranks, then restore in place from the files the
    validation opened."""
    err, d, sid = None, None, 0
    try:
        d = CheckpointDir(rank_directory(path, agent.sync.rank))
        expected = _validate(agent, mem, d.manifest)
        sid = d.manifest["save_id"]
        staging = Staging(chunk_bytes)
        d.verify(expected, staging)
    except Exception as e:   # noqa: BLE001 -- every rank must learn about every refusal
        err = e
    err = _agree(agent, err, sid)
    try:
        if err is not None:
            raise _Error(f"checkpoint {path} not loaded: {err}") from err
        _restore(agent, mem, d, staging)
    finally:
        if d is not None:
            d.close()


def _restore(agent, mem, d, staging):
    man = d.manifest
    if mem is not None:
        mem._queue = []        # the restored ring supersedes transitions queued since the save
    torch.cuda.synchronize(agent.device)
    learner = man["learner"]
    if learner["learn_stats_capacity"] != agent.learn_stats_capacity:
        agent.set_learn_stats(learner["learn_stats_capacity"])
    targets = _learner_arrays(agent)
    if mem is not None:
        targets.update(_replay_arrays(mem))
    for name, dst in targets.items():
        d.read_into(name, dst, staging)

    on, tg, opt = agent.online_net, agent.target_net, agent.optimiser
    opt.step_count.fill_(learner["optimiser_step"])
    if opt.grouped:
        opt.set_group_step_counts(learner.get("optimiser_group_steps") or [learner["optimiser_step"]] * 2)
    on.noise_seed, tg.noise_seed = learner["online_noise_seed"], learner["target_noise_seed"]
    on._noise_pending, tg._noise_pending = learner["online_noise_pending"], False
    # the saved epsilon buffers come with their stale flag: the library head reads them without launching a pending draw
    # (DESIGN.md §4), so marking them stale here would make that path draw one update early
    on._eps_stale, tg._eps_stale = learner["online_eps_stale"], learner["target_eps_stale"]
    agent._learn_calls = learner["learn_calls"]
    agent.reset_count = learner.get("reset_count") or 0
    agent.redo_count = learner.get("redo_count") or 0
    if learner.get("reset_seed") is not None:
        agent.reset_seed = learner["reset_seed"]
    if agent._horizon is not None:
        agent._horizon.set_step(learner.get("horizon_step") or 0)
    if agent._stats is not None:
        agent._stats["read"], agent._stats["last"] = learner["learn_stats_read"], None
    if mem is not None:
        rp, tr = man["replay"], mem.transitions
        for k, role in PERSISTENT_ROLES:
            if role == "state":
                setattr(mem, k, rp[k])
        tr.index, tr.full = rp["index"], rp["full"]
    torch.cuda.synchronize(agent.device)
