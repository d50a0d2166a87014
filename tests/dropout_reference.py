"""Exact NumPy models of the library's dropout masks, one per kernel family (DESIGN.md, "Dropout masks").

Every model maps element coordinates to the float32 scale the kernel multiplies by: 0 (dropped) or
float32(1) / (float32(1) - float32(p)) (kept), reproducing the kernels' float32 arithmetic bit for bit.  Element indices
are flat indices into the tensor the kernel writes ([B][T][C][W] for the time convolution, [rows][half] for GLU,
[M][N] for the GEMM, the flat buffer for w2l_act_fwd).  All functions are vectorised over uint64 arrays.

  simt_scale        dropout_scale (common.cuh): SIMT conv forward, w2l_act_fwd, GLU scalar path
  conv_mma_scale    mma.sync conv forward (TF32 and 3xTF32): the same bits, rebuilt by lane pairs
  glu_vec_scale     GLU float4 path (keep4): the same bits, one Philox block per 4 channels
  gemm_scale        GEMM epilogue: one 32-bit murmur3-style hash per pair of columns, 16 bits per element
"""
import numpy as np

MASK32 = np.uint64(0xFFFFFFFF)
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)

# fl_compat's per-call seeds: a process-global counter starting at 0x5eed0000, stepped by 0x9E3779B97F4A7C15 (mod 2^64)
FIRST_SEED = 0x5EED0000
SEED_STEP = 0x9E3779B97F4A7C15


def host_seed(k):
    """the k-th value nextSeed() returns (k = 0 is the first call)"""
    return (FIRST_SEED + k * SEED_STEP) % (1 << 64)


def _u64(x):
    return np.asarray(x, dtype=np.uint64)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 with the round structure of common.cuh's philox4x32 (which fixes c2 = c3 = 0)."""
    c0, c1, c2, c3, k0, k1 = np.broadcast_arrays(*(_u64(v) for v in (c0, c1, c2, c3, k0, k1)))
    for _ in range(10):
        p0, p1 = _M0 * c0, _M1 * c2  # 32 x 32 -> 64-bit products
        hi0, lo0 = p0 >> np.uint64(32), p0 & MASK32
        hi1, lo1 = p1 >> np.uint64(32), p1 & MASK32
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + _W0) & MASK32, (k1 + _W1) & MASK32
    return tuple(v.astype(np.uint32) for v in (c0, c1, c2, c3))


def _key(seed):
    s = _u64(seed)
    return s & MASK32, s >> np.uint64(32)


def _word(r, sel):
    return np.choose(np.asarray(sel).astype(np.intp), r)


def keep_scale(p):
    return np.float32(1) / (np.float32(1) - np.float32(p))


def _scale(keep, p):
    return np.where(keep, keep_scale(p), np.float32(0)).astype(np.float32)


def _keep24(v, p):
    """keep iff (v >> 8) * 2^-24 >= p, compared in float32"""
    return (v >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0) >= np.float32(p)


def thresh16(p):
    """the 16-bit threshold uint32(float32(p) * 65536) of the GEMM mask"""
    return np.uint32(int(np.float32(p) * np.float32(65536.0)))


def _philox_flat_bits(seed, e):
    e = _u64(e)
    k0, k1 = _key(seed)
    r = philox4x32_10((e >> np.uint64(2)) & MASK32, e >> np.uint64(34), 0, 0, k0, k1)
    return _word(r, e & np.uint64(3))


def simt_scale(seed, e, p):
    """dropout_scale: counter (e >> 2, e >> 34), key (seed lo, seed hi), word e & 3; keep iff 24 bits >= p"""
    return _scale(_keep24(_philox_flat_bits(seed, e), p), p)


def conv_mma_scale(seed, e, p, W):
    """mma.sync conv epilogue.  Lane t4 of a quad holds columns 2 t4, 2 t4 + 1 of an 8-column tile whose first element
    index `base` is a multiple of 8 (W % 8 == 0): the even lane of a pair draws the block of tile j, the odd lane that of
    tile j + 1, and they swap words, so element e ends up with word e & 3 of block e >> 2 -- dropout_scale's bits."""
    assert W % 8 == 0
    e = _u64(e)
    tile_base = e - (e & np.uint64(7))  # base + 8 j: first element of the 8-column tile
    block = (tile_base + (e & np.uint64(4))) >> np.uint64(2)  # lanes t4 = 0, 1 -> block base/4; t4 = 2, 3 -> base/4 + 1
    k0, k1 = _key(seed)
    r = philox4x32_10(block & MASK32, block >> np.uint64(32), 0, 0, k0, k1)
    return _scale(_keep24(_word(r, e & np.uint64(3)), p), p)


def glu_vec_scale(seed, e, p, H):
    """keep4: thread q of the float4 path covers elements 4q .. 4q + 3 of y [rows][H] (H % 4 == 0) with block
    (4q) >> 2 = q, words x, y, z, w in channel order"""
    assert H % 4 == 0
    e = _u64(e)
    q = e >> np.uint64(2)
    k0, k1 = _key(seed)
    r = philox4x32_10(q & MASK32, (np.uint64(4) * q) >> np.uint64(34), 0, 0, k0, k1)
    return _scale(_keep24(_word(r, e - np.uint64(4) * q), p), p)


def gemm_scale(seed, e, p):
    """GEMM epilogue, C [M][N] (N % 4 == 0), e = row N + col: idx = e >> 1 (one hash per pair of columns),
    h = ((idx lo ^ seed lo) * 0x9E3779B1 + (idx hi ^ seed hi)) mod 2^32, then the murmur3 fmix32 finaliser; element e
    takes bits 16 (e & 1) .. + 15; keep iff those 16 bits >= uint32(float32(p) * 65536)"""
    e = _u64(e)
    idx = e >> np.uint64(1)
    s_lo, s_hi = _key(seed)
    h = (((idx & MASK32) ^ s_lo) * np.uint64(0x9E3779B1) + ((idx >> np.uint64(32)) ^ s_hi)) & MASK32
    h ^= h >> np.uint64(15)
    h = (h * np.uint64(0x85EBCA77)) & MASK32
    h ^= h >> np.uint64(13)
    h = (h * np.uint64(0xC2B2AE3D)) & MASK32
    h ^= h >> np.uint64(16)
    bits = (h >> (np.uint64(16) * (e & np.uint64(1)))) & np.uint64(0xFFFF)
    return _scale(bits >= np.uint64(thresh16(p)), p)


def keep_probability(model, p):
    """exact keep probability of a model's threshold on uniform random bits"""
    p32 = np.float32(p)
    if model in (simt_scale, conv_mma_scale, glu_vec_scale):
        # smallest 24-bit value v with float32(v) * 2^-24 >= p32 (exact: v < 2^24)
        first = int(np.ceil(np.float64(p32) * 16777216.0))
        return (16777216 - first) / 16777216.0
    return (65536 - int(thresh16(p))) / 65536.0
