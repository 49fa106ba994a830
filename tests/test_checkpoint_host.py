"""The host part of rainbow_b200/checkpoint.py, without a GPU: `.npy` round trips through the bounded staging buffer across
chunk boundaries, checksum and manifest validation, refusal of object arrays and pickles, and the atomic directory rename."""
import json
import os
import pickle

import numpy as np
import pytest
import torch

from rainbow_b200 import RainbowB200Error
from rainbow_b200 import checkpoint as ck

CHUNK = 64


def staging():
    return ck.Staging(CHUNK, pin=False)


def verify(path, entry, st):
    with open(path, "rb") as f:
        ck.verify_array(f, entry, st)


def read_into(path, entry, dst, st):
    with open(path, "rb") as f:
        ck.read_array_into(f, entry, dst, st)


def reseal(directory, man):
    """Write an edited manifest with a matching digest (as a genuine writer of those values would)."""
    man = dict(man)
    man["digest"] = ck._digest(man)
    json.dump(man, open(os.path.join(directory, ck.MANIFEST), "w"))


# (chunks, elements more or less): 0 bytes, one chunk exactly, one chunk -/+ one element, several chunks (+ one)
SIZES = [(0, 0), (1, 0), (1, -1), (1, 1), (3, 0), (3, 1)]


@pytest.mark.parametrize("chunks,delta", SIZES, ids=[f"{c}chunks{d:+d}" for c, d in SIZES])
@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32, torch.int64], ids=["u8", "f32", "i64"])
def test_array_round_trip_across_chunks(tmp_path, chunks, delta, dtype):
    item = torch.empty(0, dtype=dtype).element_size()
    n = chunks * CHUNK // item + delta
    nbytes = n * item
    raw = np.random.RandomState(nbytes).randint(0, 255, nbytes).astype(np.uint8)
    src = torch.from_numpy(raw.view(np.dtype(str(dtype).split(".")[1])).copy())
    path = str(tmp_path / "a.npy")
    st = staging()
    entry = ck.write_array(path, src, st)
    assert entry["dtype"] == np.dtype(str(dtype).split(".")[1]).str and entry["shape"] == [n]
    back = np.load(path, allow_pickle=False)          # a plain .npy file any numpy reads
    assert back.tobytes() == src.numpy().tobytes()
    verify(path, entry, st)
    dst = torch.full_like(src, 7) if n else torch.empty_like(src)
    read_into(path, entry, dst, st)
    assert dst.numpy().tobytes() == src.numpy().tobytes()     # random bytes: NaN payloads included


def test_multidimensional_and_slices(tmp_path):
    st = staging()
    a = torch.arange(5 * 7 * 3, dtype=torch.float32).reshape(5, 7, 3)
    e = ck.write_array(str(tmp_path / "a.npy"), a, st)
    assert e["shape"] == [5, 7, 3]
    dst = torch.zeros(5, 7, 3)
    read_into(str(tmp_path / "a.npy"), e, dst, st)
    assert torch.equal(dst, a)
    ring = torch.arange(5, dtype=torch.int64)
    e = ck.write_array(str(tmp_path / "r.npy"), ring[:4], st)     # a leading slice, as ring_state[0:4]
    dst = torch.full((5,), -1, dtype=torch.int64)
    read_into(str(tmp_path / "r.npy"), e, dst[:4], st)
    assert dst.tolist() == [0, 1, 2, 3, -1]


def test_checksum_and_header_are_checked(tmp_path):
    st = staging()
    src = torch.arange(100, dtype=torch.float32)
    path = str(tmp_path / "a.npy")
    entry = ck.write_array(path, src, st)
    raw = bytearray(open(path, "rb").read())
    raw[-13] ^= 0x10                                    # one flipped bit in the data
    open(path, "wb").write(bytes(raw))
    with pytest.raises(RainbowB200Error, match="SHA-256"):
        verify(path, entry, st)
    open(path, "wb").write(bytes(raw[:-9]))            # truncated
    with pytest.raises(RainbowB200Error):
        verify(path, entry, st)
    ck.write_array(str(tmp_path / "b.npy"), src[:99], st)
    with pytest.raises(RainbowB200Error, match="manifest says"):
        verify(str(tmp_path / "b.npy"), entry, st)  # a different shape than the manifest entry
    e64 = ck.write_array(str(tmp_path / "c.npy"), src.double(), st)
    with pytest.raises(RainbowB200Error, match="manifest says"):
        verify(str(tmp_path / "c.npy"), entry, st)
    verify(str(tmp_path / "c.npy"), e64, st)


def test_object_arrays_and_pickles_are_refused(tmp_path):
    st = staging()
    with pytest.raises(RainbowB200Error, match="object"):
        ck.write_array(str(tmp_path / "o.npy"), np.array([{"a": 1}, None], dtype=object), st)
    assert not os.path.exists(tmp_path / "o.npy")
    np.save(tmp_path / "p.npy", np.array([{"a": 1}], dtype=object), allow_pickle=True)
    with pytest.raises(RainbowB200Error):
        verify(str(tmp_path / "p.npy"), dict(dtype="|O", shape=[1], sha256=""), st)
    with open(tmp_path / "q.npy", "wb") as f:
        pickle.dump(np.zeros(3), f)
    with pytest.raises(RainbowB200Error):
        verify(str(tmp_path / "q.npy"), dict(dtype="<f8", shape=[3], sha256=""), st)


def _dir(tmp_path, name="ck"):
    arrays = {"x": torch.arange(10, dtype=torch.int32), "y": np.linspace(0, 1, 200).astype(np.float32)}
    final = str(tmp_path / name)
    ck.write_dir(final, arrays, dict(note="hello"), chunk_bytes=CHUNK)
    return final, arrays


def test_manifest_validation(tmp_path):
    final, arrays = _dir(tmp_path)
    man = ck.read_manifest(final)
    assert man["format"] == ck.FORMAT and man["version"] == ck.VERSION and man["note"] == "hello"
    expected = {"x": ("<i4", [10]), "y": ("<f4", [200])}
    with ck.CheckpointDir(final) as d:
        d.verify(expected, staging())
        with pytest.raises(RainbowB200Error, match="missing"):
            d.verify(dict(expected, z=("<f4", [1])), staging())
        with pytest.raises(RainbowB200Error, match="needs"):
            d.verify(dict(expected, y=("<f4", [201])), staging())
    mpath = os.path.join(final, ck.MANIFEST)
    json.dump(dict(man, note="edited"), open(mpath, "w"))      # any edit without a matching digest
    with pytest.raises(RainbowB200Error, match="digest"):
        ck.read_manifest(final)
    reseal(final, dict(man, version=ck.VERSION + 1))
    with pytest.raises(RainbowB200Error, match="version"):
        ck.read_manifest(final)
    # the file name comes from the format's naming rule, never from the manifest
    bad = dict(man, arrays=dict(man["arrays"], y=dict(man["arrays"]["y"], file="../elsewhere/y.npy")))
    reseal(final, bad)
    with ck.CheckpointDir(final) as d, pytest.raises(RainbowB200Error, match="naming rule"):
        d.verify(expected, staging())
    reseal(final, man)
    os.remove(os.path.join(final, "y.npy"))
    with ck.CheckpointDir(final) as d, pytest.raises(RainbowB200Error, match="missing"):
        d.verify(expected, staging())
    open(mpath, "w").write("{not json")
    with pytest.raises(RainbowB200Error, match="manifest"):
        ck.read_manifest(final)
    with pytest.raises(RainbowB200Error, match="no checkpoint directory"):
        ck.read_manifest(str(tmp_path / "nowhere"))


def test_restore_reads_the_files_it_verified(tmp_path):
    """A newer save renamed into place between the verifying and the restoring read does not leak into the load."""
    final, arrays = _dir(tmp_path)
    with ck.CheckpointDir(final) as d:
        d.verify({"x": ("<i4", [10]), "y": ("<f4", [200])}, staging())
        ck.write_dir(final, {"x": torch.full((10,), 99, dtype=torch.int32), "y": torch.zeros(200)}, dict(note="newer"),
                     chunk_bytes=CHUNK)
        assert ck.read_manifest(final)["note"] == "newer"
        dst = torch.zeros(10, dtype=torch.int32)
        d.read_into("x", dst, staging())
    assert torch.equal(dst, arrays["x"])


def test_interrupted_replacement_falls_back_to_the_previous_directory(tmp_path):
    root = tmp_path / "ck"
    root.mkdir()
    ck.write_dir(str(root / "rank0"), {"x": torch.arange(3)}, dict(note="first"), chunk_bytes=CHUNK)
    assert ck.rank_directory(str(root), 0) == str(root / "rank0")
    os.rename(root / "rank0", root / ".rank0.old-deadbeef")      # killed between write_dir's two renames
    os.mkdir(root / ".rank0.partial-1-cafe")                      # (a partial directory is never used)
    assert ck.rank_directory(str(root), 0) == str(root / ".rank0.old-deadbeef")
    assert ck.read_manifest(ck.rank_directory(str(root), 0))["note"] == "first"
    assert ck.rank_directory(str(root), 1) == str(root / "rank1")


def test_directory_is_renamed_into_place(tmp_path, monkeypatch):
    final, _ = _dir(tmp_path)
    first = ck.read_manifest(final)
    assert sorted(os.listdir(tmp_path)) == ["ck"], "no temporary directory left behind"
    # a write that fails after its first array: the complete directory stays as it was, no partial one appears
    real, calls = ck.write_array, []

    def failing(path, src, st):
        if calls:
            raise OSError("disk full")
        calls.append(path)
        return real(path, src, st)

    monkeypatch.setattr(ck, "write_array", failing)
    with pytest.raises(OSError):
        ck.write_dir(final, {"x": torch.zeros(3), "y": torch.zeros(4)}, dict(note="second"), chunk_bytes=CHUNK)
    assert calls and os.path.dirname(calls[0]) != final, "arrays go to a temporary sibling"
    assert sorted(os.listdir(tmp_path)) == ["ck"]
    assert ck.read_manifest(final) == first
    with pytest.raises(OSError):
        ck.write_dir(str(tmp_path / "other"), {"x": torch.zeros(3), "y": torch.zeros(4)}, {}, chunk_bytes=CHUNK)
    assert sorted(os.listdir(tmp_path)) == ["ck"]
    monkeypatch.setattr(ck, "write_array", real)
    # a complete second write replaces the first
    ck.write_dir(final, {"x": torch.ones(2)}, dict(note="third"), chunk_bytes=CHUNK)
    assert ck.read_manifest(final)["note"] == "third" and sorted(os.listdir(final)) == [ck.MANIFEST, "x.npy"]
    assert sorted(os.listdir(tmp_path)) == ["ck"]
