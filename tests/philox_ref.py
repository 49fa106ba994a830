"""numpy references of the random-shift augmentation (rb_gather_shift): Philox4x32-10 (Salmon et al. 2011, the Random123
construction the device code implements in rainbow_b200/csrc/rb_internal.cuh), the offsets drawn from it, and the shift
itself as ReplicationPad2d(pad) followed by an 84 x 84 crop.  Also the two uniforms box_muller forms from a pair of
Philox words, which the intensity (drq_ref) and noise (noise_ref) references share."""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
SHIFT_STREAM = 0x53484654
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: uint32 [..., 4], key: uint32 [..., 2] (broadcast) -> uint32 [..., 4]."""
    c = [np.asarray(ctr, dtype=np.uint32)[..., i].astype(np.uint64) for i in range(4)]
    k = np.asarray(key, dtype=np.uint32).astype(np.uint64)
    k0, k1 = k[..., 0], k[..., 1]
    for _ in range(10):
        p0, p1 = M0 * c[0], M1 * c[2]
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & _LO, p1 >> np.uint64(32), p1 & _LO
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0, k1 = (k0 + W0) & _LO, (k1 + W1) & _LO
    return np.stack([x.astype(np.uint32) for x in c], axis=-1)


def box_muller_uniforms(a, b):
    """float64 (u1, u2) of box_muller (rb_internal.cuh) for words a, b: u1 = fl32(fl32(a) + 1) 2^-32 in (0, 1] and
    u2 = fl32(b) 2^-32 in [0, 1), the device's exact fp32 values (scaling by 2^-32 is exact)."""
    u1 = (np.asarray(a).astype(np.float32) + np.float32(1.0)).astype(np.float64) * 2.0 ** -32
    u2 = np.asarray(b).astype(np.float32).astype(np.float64) * 2.0 ** -32
    return u1, u2


def shift_offsets(seed, counter, B, pad):
    """int32 [2][B][2] -- (side: 0 state, 1 next state; sample; (oy, ox)) -- as rb_gather_shift draws them for the replay
    seed and the value of its rng_counter the gather reads."""
    b = np.arange(B, dtype=np.uint64)
    ctr = np.stack([np.full(B, counter & 0xFFFFFFFF, np.uint64), np.full(B, (counter >> 32) & 0xFFFFFFFF, np.uint64), b,
                    np.full(B, SHIFT_STREAM, np.uint64)], axis=-1).astype(np.uint32)
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], dtype=np.uint32)
    words = philox4x32_10(ctr, key).astype(np.uint64)
    off = ((words * np.uint64(2 * pad + 1)) >> np.uint64(32)).astype(np.int32)   # [B, 4]
    return np.stack([off[:, 0:2], off[:, 2:4]])


def shift_ref(x, offsets, pad):
    """x: [B, C, 84, 84], offsets: int [B, 2] (oy, ox) in [0, 2 pad] -> np.pad(mode="edge") by pad, then the 84 x 84 crop
    at (oy, ox) of each sample."""
    B, C, H, W = x.shape
    padded = np.pad(x, ((0, 0), (0, 0), (pad, pad), (pad, pad)), mode="edge")
    rows = offsets[:, 0, None] + np.arange(H)            # [B, H]
    cols = offsets[:, 1, None] + np.arange(W)            # [B, W]
    return padded[np.arange(B)[:, None, None, None], np.arange(C)[None, :, None, None], rows[:, None, :, None],
                  cols[:, None, None, :]]
