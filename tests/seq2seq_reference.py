"""Exact NumPy models of the Seq2Seq criterion's random draws (csrc/seq2seq.cu; DESIGN.md §9).

  substituted_tokens   the decoder's input tokens under teacher forcing with substitution (--pctteacherforcing < 100)
  dropout_scales       the scale after GRU layer k of the flattened round-major stack (w2l_act_fwd's mask, seed + 1 + k)
"""
import numpy as np

import dropout_reference as R


def substituted_tokens(seed, y, N, pct):
    """tokens [B,U]: column 0 is N (startEmbedding); tokens[b][u] = y[b][u-1] unless r1 < float32(1 - pct/100), then
    min(floor(float32(r2) * float32(N - 1)), N - 2), with r1 / r2 words x / y of Philox block (e lo, e hi) for
    e = b * U + u, each (word >> 8) * 2^-24 in float32"""
    y = np.asarray(y, np.int64)
    B, U = y.shape
    out = np.full((B, U), N, np.int64)
    out[:, 1:] = y[:, :-1]
    q = np.float32(1.0 - pct / 100.0)
    if q <= 0:
        return out
    e = np.arange(B * U, dtype=np.uint64)
    k0, k1 = R._key(seed)
    w = R.philox4x32_10(e & R.MASK32, e >> np.uint64(32), 0, 0, k0, k1)
    r1 = (w[0] >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    r2 = (w[1] >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    sub = np.minimum(np.floor(r2 * np.float32(N - 1)).astype(np.int64), N - 2)
    repl = (r1 < q).reshape(B, U)
    repl[:, 0] = False
    return np.where(repl, sub.reshape(B, U), out)


def dropout_scales(seed, k, shape, p):
    """the [B,U,H] float32 scale applied after layer k (flat element index into [B][U][H])"""
    n = int(np.prod(shape))
    return R.simt_scale((seed + 1 + k) % (1 << 64), np.arange(n, dtype=np.uint64), p).reshape(shape)
