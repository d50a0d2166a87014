"""CPU checks of the dropout mask definitions in tests/dropout_reference.py: the Philox round structure against the
Random123 known-answer vectors, keep rates, independence of the keep decisions at every index distance the kernels
exploit (neighbours, the two 16-bit halves of a word, the four words of a Philox block, one column / channel / frame
apart), across consecutive host seeds, and at element indices of 2^34 and beyond.  tests/test_gpu_dropout.py proves each
kernel equal to its model bit for bit, so these statistics hold for the kernels."""
import functools

import numpy as np
import pytest

import dropout_reference as R

# a [B][T][C][W] activation of the TDS / streaming TDS archs (C = 15, W = 80), ~1.2M elements
B, T, C, W = 2, 500, 15, 80
N = B * T * C * W

MODELS = {
    "simt": lambda s, e, p: R.simt_scale(s, e, p),
    "conv_mma": lambda s, e, p: R.conv_mma_scale(s, e, p, W),
    "glu_vec": lambda s, e, p: R.glu_vec_scale(s, e, p, W),
    "gemm": lambda s, e, p: R.gemm_scale(s, e, p),  # C [B*T*C rows][W columns]
}
BASE_MODEL = {"simt": R.simt_scale, "conv_mma": R.conv_mma_scale, "glu_vec": R.glu_vec_scale, "gemm": R.gemm_scale}
SEED = R.host_seed(3)


@functools.lru_cache(maxsize=None)
def keep(name, seed, p=0.5, offset=0):
    e = np.arange(N, dtype=np.uint64) + np.uint64(offset)
    return MODELS[name](seed, e, p) != 0


def test_philox_known_answers():
    """Random123's kat_vectors for philox4x32_10"""
    cases = [
        ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
        ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
        ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
    ]
    for ctr, key, want in cases:
        got = R.philox4x32_10(*ctr, *key)
        assert tuple(int(v) for v in got) == want, [hex(int(v)) for v in got]


def test_pinned_philox_sites_share_dropout_scale_bits():
    """the mma.sync conv and GLU float4 models, written from their kernels' index arithmetic, are dropout_scale's mask"""
    e = np.arange(N, dtype=np.uint64) + np.uint64((1 << 34) - 4000)  # crosses the high counter word
    for p in (0.2, 0.5):
        ref = R.simt_scale(SEED, e, p)
        assert np.array_equal(R.conv_mma_scale(SEED, e, p, W), ref)
        assert np.array_equal(R.glu_vec_scale(SEED, e, p, W), ref)


@pytest.mark.parametrize("name", list(MODELS))
@pytest.mark.parametrize("p", [0.1, 0.2, 0.25, 0.5, 0.590432749713])
def test_keep_rate_and_scale(name, p):
    s = MODELS[name](SEED, np.arange(N, dtype=np.uint64), p)
    assert set(np.unique(s).tolist()) <= {0.0, float(R.keep_scale(p))}
    assert s.dtype == np.float32
    q = R.keep_probability(BASE_MODEL[name], p)
    assert abs(q - (1 - p)) < 2e-5  # the 16-bit threshold's quantisation
    rate = float(np.count_nonzero(s)) / N
    sigma = np.sqrt(q * (1 - q) / N)
    assert abs(rate - q) < 5 * sigma, (name, p, rate, q, sigma)


def _corr(a, b):
    a, b = a.astype(np.float64), b.astype(np.float64)
    return float(np.corrcoef(a, b)[0, 1]), a.size


def _pairs():
    """(label, flat distance d, selector of the first element i given its coordinates) — the index distances the kernels
    exploit: neighbours, the halves of a 32-bit word, the four words of a Philox block, one column / channel / frame"""
    e = np.arange(N, dtype=np.int64)
    c = (e // W) % C
    out = [(f"neighbour {d}", d, np.ones(N, bool)) for d in (1, 2, 3, 4, 8)]
    out += [("column", 1, np.ones(N, bool)), ("channel", W, np.ones(N, bool)), ("frame", C * W, np.ones(N, bool))]
    out.append(("word halves (flat)", 1, e % 2 == 0))
    out.append(("word halves (channels)", W, c % 2 == 0))
    for a in range(4):
        for b in range(a + 1, 4):
            out.append((f"block words {a},{b} (flat)", b - a, e % 4 == a))
            out.append((f"block words {a},{b} (channels)", 2 * (b - a) * W, c % 8 == 2 * a))
    return out


@pytest.mark.parametrize("name", list(MODELS))
def test_keep_decisions_are_uncorrelated_at_kernel_distances(name):
    k = keep(name, SEED)
    bad = []
    for label, d, sel in _pairs():
        i = np.nonzero(sel[: N - d])[0]
        r, n = _corr(k[i], k[i + d])
        if abs(r) >= 5 / np.sqrt(n):
            bad.append((label, r, n))
    assert not bad, (name, bad)


@pytest.mark.parametrize("name", list(MODELS))
def test_consecutive_host_seeds_are_independent(name):
    for j in range(3):
        a, b = keep(name, R.host_seed(j)), keep(name, R.host_seed(j + 1))
        r, n = _corr(a, b)
        assert abs(r) < 5 / np.sqrt(n), (name, j, r)
        # and no shifted copy of each other at the kernels' distances
        for d in (1, 2, 4, W):
            r, n = _corr(a[:-d], b[d:])
            assert abs(r) < 5 / np.sqrt(n), (name, j, d, r)


@pytest.mark.parametrize("name", list(MODELS))
@pytest.mark.parametrize("high", [1 << 32, 1 << 34, 1 << 35, (1 << 34) * 3 + (1 << 33)])
def test_high_indices_do_not_alias_low_ones(name, high):
    lo, hi = keep(name, SEED), keep(name, SEED, offset=high)
    assert not np.array_equal(lo, hi)
    r, n = _corr(lo, hi)
    assert abs(r) < 5 / np.sqrt(n), (name, high, r)
