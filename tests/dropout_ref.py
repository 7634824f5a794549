"""Host statement of the dropout rule of include/speecht5_b200.h (lines 16-18), for checking kernels' masks exactly.

Philox4x32-7(seed, offset, i / 8) -> four 32-bit words = eight 16-bit lanes; element i is kept iff lane i % 8 is
>= drop_threshold(p). Counter words: c0, c1 = low / high word of i / 8, c2, c3 = low / high word of `offset`; key words
k0, k1 = low / high word of `seed` (csrc/ptx.cuh philox4x32, philox_lane16; csrc/kernels.cuh drop_threshold).
Attention probabilities use the row index prow = (b * H + h) * Tq + i and a row pitch of Tk rounded up to 32 keys.
Vectorised numpy: uint64 arithmetic masked to 32 bits."""
import numpy as np

ROUNDS = 7
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_LO = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)


def philox4x32(seed, offset, ctr):
    """(x, y, z, w) uint64 arrays (values < 2^32) of Philox4x32-7 at counter `ctr` (scalar or array)."""
    ctr = np.asarray(ctr, dtype=np.uint64)
    seed, offset = int(seed) & (2**64 - 1), int(offset) & (2**64 - 1)
    k0, k1 = seed & 0xFFFFFFFF, seed >> 32
    c0 = ctr & _LO
    c1 = ctr >> _S32
    c2 = np.full_like(ctr, offset & 0xFFFFFFFF)
    c3 = np.full_like(ctr, offset >> 32)
    for _ in range(ROUNDS):
        p0 = _M0 * c0  # < 2^64: exact in uint64
        p1 = _M1 * c2
        h0, l0 = p0 >> _S32, p0 & _LO
        h1, l1 = p1 >> _S32, p1 & _LO
        c0, c1, c2, c3 = h1 ^ c1 ^ np.uint64(k0), l1, h0 ^ c3 ^ np.uint64(k1), l0
        k0 = (k0 + _W0) & 0xFFFFFFFF
        k1 = (k1 + _W1) & 0xFFFFFFFF
    return c0, c1, c2, c3


def drop_threshold(p):
    """16-bit keep threshold: p * 65536 evaluated in fp32, truncated, clamped to 65535; 0 for p <= 0 (no dropout)."""
    p32 = np.float32(p)
    if p32 <= 0:
        return 0
    t = np.float32(p32 * np.float32(65536.0))
    return 65535 if t >= np.float32(65535.0) else int(t)


def drop_scale(p):
    """The factor kept elements are multiplied by: 1 / (1 - p) in fp32 (1 without dropout)."""
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(p))) if p > 0 else 1.0


def lanes16(seed, offset, idx):
    """The 16-bit Philox lane that decides element idx (uint64 array)."""
    idx = np.asarray(idx, dtype=np.uint64)
    x, y, z, w = philox4x32(seed, offset, idx >> np.uint64(3))
    lane = (idx & np.uint64(7)).astype(np.int64)
    word = np.choose(lane >> 1, (x, y, z, w))
    return np.where((lane & 1) == 1, word >> np.uint64(16), word & np.uint64(0xFFFF))


def keep_mask(seed, offset, idx, p):
    """bool array: True where element idx (logical index, any shape) survives dropout with probability p."""
    idx = np.asarray(idx, dtype=np.uint64)
    thr = drop_threshold(p)
    if thr == 0:
        return np.ones(idx.shape, dtype=bool)
    return lanes16(seed, offset, idx) >= np.uint64(thr)


def attn_pitch(Tk):
    """Row pitch of the attention dropout index: Tk rounded up to a multiple of 32 keys."""
    return (int(Tk) + 31) & ~31


def attn_index(b, h, i, j, H, Tq, Tk):
    """Dropout index of probability (b, h, i, j): ((b * H + h) * Tq + i) * attn_pitch(Tk) + j (broadcasting)."""
    b, h, i, j = (np.asarray(t, dtype=np.uint64) for t in (b, h, i, j))
    prow = (b * np.uint64(H) + h) * np.uint64(Tq) + i
    return prow * np.uint64(attn_pitch(Tk)) + j


def attn_keep(seed, offset, p, B, H, Tq, Tk):
    """[B, H, Tq, Tk] keep mask of attention probabilities."""
    b, h, i, j = np.ix_(np.arange(B), np.arange(H), np.arange(Tq), np.arange(Tk))
    return keep_mask(seed, offset, attn_index(b, h, i, j, H, Tq, Tk), p)
