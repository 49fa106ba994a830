"""CPU tests of the random-shift augmentation's references and host side: the numpy Philox4x32-10 of tests/philox_ref.py
against Random123's known-answer vectors, the numpy shift against the formula it stands for, the offsets' range, and
rb_gather_shift's argument refusals through the built library (answered before any launch, so no GPU is needed)."""
import numpy as np
import pytest

import philox_ref as P


@pytest.mark.parametrize("ctr,key,want", [
    ([0, 0, 0, 0], [0, 0], [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]),
    ([0xFFFFFFFF] * 4, [0xFFFFFFFF, 0xFFFFFFFF], [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]),
    ([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], [0xA4093822, 0x299F31D0],
     [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]),
], ids=["zero", "ones", "pi"])
def test_philox_known_answers(ctr, key, want):
    got = P.philox4x32_10(np.array(ctr, np.uint32), np.array(key, np.uint32))
    assert got.dtype == np.uint32 and got.tolist() == want
    batch = P.philox4x32_10(np.array([ctr, ctr], np.uint32), np.array(key, np.uint32))   # broadcast over counters
    assert batch.tolist() == [want, want]


def loop_shift(x, offsets, pad):
    """The formula itself: out[c][y][x] = in[c][clamp(y + oy - pad)][clamp(x + ox - pad)]."""
    B, C, H, W = x.shape
    out = np.empty_like(x)
    for b in range(B):
        oy, ox = offsets[b]
        for y in range(H):
            for xx in range(W):
                out[b, :, y, xx] = x[b, :, min(max(y + oy - pad, 0), H - 1), min(max(xx + ox - pad, 0), W - 1)]
    return out


@pytest.mark.parametrize("pad", [1, 4, 16])
def test_shift_reference_is_pad_then_crop(pad):
    rs = np.random.RandomState(pad)
    x = rs.rand(5, 2, 84, 84).astype(np.float32)
    offsets = rs.randint(0, 2 * pad + 1, (5, 2)).astype(np.int32)
    offsets[0], offsets[1], offsets[2] = (0, 0), (2 * pad, 2 * pad), (pad, pad)     # both corners and the identity
    got = P.shift_ref(x, offsets, pad)
    assert np.array_equal(got, loop_shift(x, offsets, pad))
    assert np.array_equal(got[2], x[2])
    # the corner crops replicate the first / last row and column pad times
    assert np.array_equal(got[0, :, :pad + 1, 0], np.repeat(x[0, :, :1, 0], pad + 1, axis=1))
    assert np.array_equal(got[1, :, -pad - 1:, -1], np.repeat(x[1, :, -1:, -1], pad + 1, axis=1))


@pytest.mark.parametrize("pad", [1, 4, 16])
def test_offsets_cover_exactly_the_range(pad):
    off = P.shift_offsets(0x0123456789ABCDEF, (5 << 32) + 17, 4096, pad)
    assert off.shape == (2, 4096, 2) and off.dtype == np.int32
    assert off.min() == 0 and off.max() == 2 * pad
    assert not np.array_equal(off[0], off[1]), "state and next state draw their own offsets"
    again = P.shift_offsets(0x0123456789ABCDEF, (5 << 32) + 18, 4096, pad)
    assert not np.array_equal(off, again), "the counter changes the draws"
    # words x, y -> state, z, w -> next state, from one Philox call keyed by the seed
    w = P.philox4x32_10(np.array([17, 5, 3, P.SHIFT_STREAM], np.uint32), np.array([0x89ABCDEF, 0x01234567], np.uint32))
    want = [int((int(v) * (2 * pad + 1)) >> 32) for v in w]
    assert off[:, 3].reshape(-1).tolist() == want


def test_gather_shift_refusals_without_gpu():
    from rainbow_b200 import _lib
    lib = _lib.load()
    one = 8   # never dereferenced: validation fails first
    # frames, timestep, action, reward, nonterminal, size, data_idx, B, history, n, gamma_pow, states, next_states, actions,
    # returns, nonterminals, pad, seed, rng_counter, shifts, stream
    good = [one] * 5 + [1000, one, 32, 4, 3] + [one] * 6 + [4, 7, one, one, None]
    ptrs = [0, 1, 2, 3, 4, 6, 10, 11, 12, 13, 14, 15, 18, 19]

    def call(**change):
        a = list(good)
        for i, v in change.items():
            a[int(i[1:])] = v
        return lib.rb_gather_shift(*a)

    for i in ptrs:
        assert call(**{f"a{i}": None}) == -22, i
        assert b"null" in lib.rb_last_error()
    for pad in (0, -1, 17, 1000):
        assert call(a16=pad) == -34, pad
    assert call(a8=40, a9=30) == -34            # window > RB_MAX_WINDOW (rb_gather's check)
    assert call(a7=65536) == -34                # B > 65535
    for i, v in ((7, 0), (8, 0), (9, 0), (5, 0)):
        assert call(**{f"a{i}": v}) == -22, i   # sizes must be positive
    assert lib.rb_gather(one, one, one, one, one, 8, one, 4, 40, 30, one, one, one, one, one, one, None) == -34


def test_kernel_id_and_signature():
    from rainbow_b200 import _lib
    assert _lib.KERNEL_IDS[-1] == "gather_shift" and _lib.KERNEL_IDS.index("gather") == 3
    assert len(_lib.SIGNATURES["rb_gather_shift"][1]) == 21


def test_invalid_pad_and_numpy_stream_refused_before_cuda():
    """The replay checks shift_pad before it touches the device; Agent's check runs at construction (GPU tests)."""
    from rainbow_b200.memory import ReplayMemory
    mem = ReplayMemory.__new__(ReplayMemory)      # host fields only: the checks need nothing else
    mem.rng = "philox"
    assert mem._check_shift_pad(0) == 0 and mem._check_shift_pad(16) == 16
    for bad in (-1, 17):
        with pytest.raises(ValueError):
            mem._check_shift_pad(bad)
    mem.rng = "numpy"
    assert mem._check_shift_pad(0) == 0
    with pytest.raises(ValueError):
        mem._check_shift_pad(4)
