"""The float64 beam search of tests/seq2seq_beam_reference.py (DESIGN.md §9) on synthetic log-prob tables: against
brute-force enumeration, each rule of the walk on hand-built tables, and K = 1 against the greedy decode."""
import itertools

import numpy as np
import pytest
import torch

import seq2seq_beam_reference as beamref
from oracle import seq2seq_ref as ref


def table_step(fn):
    """(step, init) over a table: fn(prefix tuple) -> log-probs [N]"""
    def step(prefix):
        return np.asarray(fn(prefix), np.float64), lambda t: prefix + (t,)
    return step, ()


def random_table(N, seed):
    rng = np.random.default_rng(seed)
    cache = {}

    def fn(prefix):
        if prefix not in cache:
            cache[prefix] = np.log(rng.dirichlet(np.ones(N)))
        return cache[prefix]
    return fn


def hand_table(rows, default):
    return lambda prefix: np.asarray(rows.get(prefix, default), np.float64)


@pytest.mark.parametrize("N,maxlen,seed", [(3, 4, 0), (3, 4, 1), (4, 3, 2)])
def test_against_enumeration(N, maxlen, seed):
    """K larger than every beam the search can hold: nothing is pruned, no cap applies, so the search returns every
    eos-terminated sequence shorter than maxlen, in completion order: by length, then by score"""
    eos = N - 2
    fn = random_table(N, seed)
    K = 64  # above the candidates of any step: (N - 1)^(maxlen - 1) N <= 36
    hyps, _ = beamref.beam(*table_step(fn), K, maxlen, eos)
    want = []
    for length in range(maxlen):
        group = []
        for path in itertools.product([c for c in range(N) if c != eos], repeat=length):
            s = sum(fn(path[:i])[path[i]] for i in range(length)) + fn(path)[eos]
            group.append((s, list(path)))
        want += sorted(group, key=lambda e: -e[0])
    assert len(want) < K
    assert [p for _, p in hyps] == [p for _, p in want]
    np.testing.assert_allclose([s for s, _ in hyps], [s for s, _ in want], rtol=0, atol=1e-12)


def test_eos_at_rank_k_or_beyond_is_dropped():
    # K = 2, eos = 2.  Step 0: beam [0] (-1), [1] (-1.5).  Step 1 ranks: [0,0] -1.5 (extends), [0]+eos -2.05 (rank 1:
    # completes), [1]+eos -2.1 (rank 2 >= K: dropped), [0,1] -5 (extends, the beam is full)
    t = hand_table({(): [-1, -1.5, -9, -9], (0,): [-0.5, -4, -1.05, -9], (1,): [-9, -9, -0.6, -9]}, [-9, -9, -9, -9])
    hyps, _ = beamref.beam(*table_step(t), 2, 2, 2)
    assert [p for _, p in hyps] == [[0]]
    assert hyps[0][0] == pytest.approx(-2.05)


def test_k_cap_sorts_and_early_stop():
    # K = 2.  Step 0: [0] -1 (extends), [] -1.1 (completes), [1] -9 (extends).  Step 1: [0]+eos -1.05 completes first;
    # two completions: the cap sorts them ([0] before []), and the second (-1.1) beats the best live score (-6): stop
    t = hand_table({(): [-1, -9, -1.1, -9], (0,): [-5, -5, -0.05, -5]}, [-1, -1, -50, -1])
    hyps, _ = beamref.beam(*table_step(t), 2, 10, 2)
    assert [p for _, p in hyps] == [[0], []]
    np.testing.assert_allclose([s for s, _ in hyps], [-1.05, -1.1])


def test_k_cap_drops_the_worst():
    # K = 2: step 0 completes [] (-2) at rank 1; step 1 completes [0] (-1.5) at rank 1: the cap sorts [0], [], and -2
    # is not above the best live score (-1.3), so the search goes on; step 2 completes [0, 0] (-1.4): the cap keeps
    # [0, 0], [0] and drops []
    t = hand_table({(): [-0.5, -3, -2, -9], (0,): [-0.8, -9, -1.0, -9], (1,): [-9, -9, -9, -9], (0, 0): [-5, -9, -0.1, -9]},
                   [-9, -9, -9, -9])
    hyps, _ = beamref.beam(*table_step(t), 2, 5, 2)
    assert [p for _, p in hyps] == [[0, 0], [0]]
    np.testing.assert_allclose([s for s, _ in hyps], [-1.4, -1.5])


def test_early_stop_needs_the_kth_completion_above_the_best_live_score():
    # as test_k_cap_sorts_and_early_stop, but the live [0,0] scores -1.06 > -1.1: no stop, and at maxlen the
    # completions (sorted, since the cap applied) come back
    t = hand_table({(): [-1, -9, -1.1, -9], (0,): [-0.06, -5, -0.05, -5]}, [-20, -20, -30, -20])
    hyps, _ = beamref.beam(*table_step(t), 2, 2, 2)
    assert [p for _, p in hyps] == [[0], []]
    hyps3, _ = beamref.beam(*table_step(t), 2, 3, 2)
    assert [p for _, p in hyps3] == [[0], []]


def test_maxlen_without_completions_returns_the_live_beam():
    t = hand_table({}, [-1, -1.5, -50, -2])
    hyps, _ = beamref.beam(*table_step(t), 2, 4, 2)
    assert [p for _, p in hyps] == [[0, 0, 0, 0], [0, 0, 0, 1]]
    np.testing.assert_allclose([s for s, _ in hyps], [-4, -4.5])


def test_maxlen_with_fewer_than_k_completions_keeps_completion_order():
    # K = 3: [] completes at step 0 with -1.2, [0] at step 1 with -1.1 (better, but no cap: completion order)
    t = hand_table({(): [-1, -3, -1.2, -4], (0,): [-5, -6, -0.1, -7]}, [-1, -1, -60, -1])
    hyps, _ = beamref.beam(*table_step(t), 3, 3, 2)
    assert [p for _, p in hyps] == [[], [0]]
    np.testing.assert_allclose([s for s, _ in hyps], [-1.2, -1.1])


def test_beam_narrower_than_k():
    # N = 3, K = 4: step 0 has three candidates, so the beam holds two; step 1 has six
    t = hand_table({(): [-1, -2, -3]}, [-1, -2, -0.5])
    hyps, _ = beamref.beam(*table_step(t), 4, 2, 2)
    assert [p for _, p in hyps] == [[], [0], [1]]
    np.testing.assert_allclose([s for s, _ in hyps], [-3, -1.5, -2.5])


def test_k1_is_greedy():
    torch.manual_seed(0)
    N, H, Tp, R, L = 11, 16, 9, 2, 2
    params = [p.detach() for p in ref.unflatten(torch.rand(sum(int(np.prod(s)) for s in ref.param_shapes(N, H, R, L)) + 64) * 2 - 1,
                                                _layout(N, H, R, L), N, H, R, L)]
    x = torch.randn(3, Tp, 2 * H, dtype=torch.float64)
    for b, (want, _gaps) in enumerate(ref.greedy(params, x, N - 2, 12, R, L)):
        hyps, _ = beamref.beam(*beamref.model_step(params, x[b:b + 1], R, L), 1, 12, N - 2)
        assert len(hyps) == 1 and hyps[0][1] == want


def _layout(N, H, R, L):
    out, off = [], 0
    for s in ref.param_shapes(N, H, R, L):
        n = int(np.prod(s))
        out.append((off, n, s))
        off += n
    return out
