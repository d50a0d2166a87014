"""Pins for the CPU oracle above 32 tokens, where the 64-wide GPU entry points are checked against it: brute-force
enumeration of all N^T paths (N = 40 and 64, T = 3) and of all monotone alignments, as test_oracle_pins.py does for
small N."""
import itertools

import numpy as np
import pytest

import oracle


def softmax_all(s):
    m = s.max()
    w = np.exp(s - m)
    return m + np.log(w.sum()), w / w.sum()


def brute_fcc3(e, tr):
    """all N^3 paths at once: logZ, marginals [3,N], pair marginals [N,N] (to, from), best path."""
    e = e.astype(np.float64)
    tr = tr.astype(np.float64)
    N = e.shape[1]
    # s[a, b, c] = path (a, b, c)
    s = e[0][:, None, None] + e[1][None, :, None] + e[2][None, None, :] + tr.T[:, :, None] + tr.T[None, :, :]
    logz, w = softmax_all(s)
    marg = np.stack([w.sum(axis=(1, 2)), w.sum(axis=(0, 2)), w.sum(axis=(0, 1))])
    pair = w.sum(axis=2).T + w.sum(axis=0).T  # [to][from] for steps 0 -> 1 and 1 -> 2
    best = np.unravel_index(int(np.argmax(s)), (N, N, N))
    return logz, marg, pair, list(best)


def brute_fac(e, y, tr):
    e = e.astype(np.float64)
    tr = tr.astype(np.float64)
    T, N = e.shape
    L = len(y)
    scores, als = [], []
    for adv in itertools.combinations(range(1, T), L - 1):
        a, l = [], 0
        for t in range(T):
            l += t in adv
            a.append(l)
        s = e[0, y[a[0]]] + sum(e[t, y[a[t]]] + tr[y[a[t]], y[a[t - 1]]] for t in range(1, T))
        scores.append(s)
        als.append(a)
    logz, w = softmax_all(np.asarray(scores))
    marg = np.zeros((T, N))
    pair = np.zeros((N, N))
    for wi, a in zip(w, als):
        for t in range(T):
            marg[t, y[a[t]]] += wi
        for t in range(1, T):
            pair[y[a[t]], y[a[t - 1]]] += wi
    return logz, marg, pair


@pytest.mark.parametrize("N,y", [(40, [39, 5]), (40, [7, 33, 7]), (64, [63, 0]), (64, [32, 31, 32])])
def test_asg_wide_against_enumeration(N, y):
    rng = np.random.default_rng(N + len(y))
    e = rng.normal(0, 2, (1, 3, N)).astype(np.float32)
    tr = (np.eye(N) + rng.normal(0, 0.5, (N, N))).astype(np.float32)
    tgt = np.asarray([y], np.int32)
    fz, fm, fp, best = brute_fcc3(e[0], tr)
    az, am, ap = brute_fac(e[0], y, tr)
    loss, de, dt = oracle.asg(e, tgt, tr)
    np.testing.assert_allclose(loss[0], fz - az, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(de[0], fm - am, atol=1e-5)
    np.testing.assert_allclose(dt, fp - ap, atol=1e-5)
    np.testing.assert_allclose(oracle.fcc(e, tr, backward=False)[0], fz, rtol=1e-6)
    assert oracle.fcc_viterbi(e, tr)[0].tolist() == best
