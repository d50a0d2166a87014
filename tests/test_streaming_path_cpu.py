"""The carried FCC Viterbi of the streaming criterion path (tests/streaming_path_reference.py, the model of
w2l_stream_run_path for ASG / LinSeg) against the whole-utterance FCC Viterbi of the C oracle (oracle/w2l_oracle.c):

- over random chunkings, calls without frames included, the committed labels put end to end are the full Viterbi
  path, ties (first maximum) included, and each call reports the frame index of its first label;
- the convergence rule commits frames before finish when the survivors meet;
- past the pending bound the oldest frames are committed along the best path so far and counted, and nothing else is.
No GPU needed."""
import numpy as np
import pytest

import oracle
from streaming_path_reference import CarriedViterbi, tied_forever


def stream(emis, trans, chunks, max_pending=1024):
    """emis [T, N] fed in calls of `chunks` frames, then finish with no new data: (joined labels, per call (labels,
    first, forced))"""
    cv = CarriedViterbi(trans, max_pending)
    calls, t0 = [], 0
    for c in chunks:
        calls.append(cv.run(emis[t0:t0 + c]))
        t0 += c
    assert t0 == len(emis)
    calls.append(cv.run(emis[:0], finish=True))
    return np.concatenate([c[0] for c in calls]), calls


def random_chunks(rng, T):
    out = []
    while sum(out) < T:
        out.append(int(min(T - sum(out), rng.choice([0, 1, 2, 5, 13, 40]))))
    return out


def case(rng, N, T, ties):
    if ties:  # few distinct small integers: many exact ties between candidates and between end states
        emis = rng.integers(-2, 3, (T, N)).astype(np.float32)
        trans = rng.integers(-2, 3, (N, N)).astype(np.float32)
    else:
        emis = (rng.normal(0, 2, (T, N))).astype(np.float32)
        trans = (2 * np.eye(N) + rng.normal(0, 1, (N, N))).astype(np.float32)
    return emis, trans


@pytest.mark.parametrize("N", [1, 2, 5, 30, 32, 33, 64])
@pytest.mark.parametrize("ties", [False, True])
def test_joined_path_is_the_full_viterbi(N, ties):
    rng = np.random.default_rng(N * 10 + ties)
    T = 157
    emis, trans = case(rng, N, T, ties)
    full = oracle.fcc_viterbi(emis[None], trans)[0]
    for _ in range(6):
        chunks = random_chunks(rng, T)
        joined, calls = stream(emis, trans, chunks)
        np.testing.assert_array_equal(joined, full, err_msg=str(chunks))
        firsts = np.cumsum([0] + [len(c[0]) for c in calls[:-1]])
        assert [c[1] for c in calls] == firsts.tolist()
        assert all(c[2] == 0 for c in calls)


def test_converged_frames_commit_before_finish():
    rng = np.random.default_rng(3)
    N, T = 30, 200
    emis = rng.normal(0, 4, (T, N)).astype(np.float32)
    trans = rng.normal(0, 1, (N, N)).astype(np.float32)
    joined, calls = stream(emis, trans, [50] * 4)
    early = sum(len(c[0]) for c in calls[:-1])
    assert early > T // 2, early  # well-separated scores: the survivors meet a few frames back
    np.testing.assert_array_equal(joined, oracle.fcc_viterbi(emis[None], trans)[0])


@pytest.mark.parametrize("N", [2, 5])
def test_forced_commit(N):
    """states 0 and 1 stay tied and never share a predecessor, so nothing converges: every frame past the bound is
    forced, along the first-maximum state (0); the first forced prefix is the Viterbi path of the frames so far"""
    bound, T = 16, 100
    emis, trans = tied_forever(N, T)
    chunks = [7] * 14 + [2]
    joined, calls = stream(emis, trans, chunks, max_pending=bound)
    fed = np.cumsum(chunks)
    for k, (labels, first, forced) in enumerate(calls[:-1]):
        assert forced == max(0, fed[k] - bound), (k, forced)
        assert first == max(0, (fed[k - 1] if k else 0) - bound)
        assert len(labels) == forced - (max(0, fed[k - 1] - bound) if k else 0)
    first_forced = next(k for k, c in enumerate(calls) if len(c[0]))
    prefix = oracle.fcc_viterbi(emis[None, :fed[first_forced]], trans)[0]
    np.testing.assert_array_equal(calls[first_forced][0], prefix[:len(calls[first_forced][0])])
    assert calls[-1][2] == T - bound  # finish commits the rest and forces nothing
    assert len(joined) == T
    np.testing.assert_array_equal(joined, np.zeros(T, np.int32))


def test_forcing_keeps_the_bound():
    """random, nearly flat emissions under a tight bound: every call leaves at most `bound` frames pending, the calls'
    frame indices follow each other, and finish commits exactly the rest"""
    rng = np.random.default_rng(9)
    N, T, bound = 5, 300, 3
    emis = rng.normal(0, 0.002, (T, N)).astype(np.float32)
    trans = np.full((N, N), -0.01, np.float32)  # each state prefers its own past: the survivors meet late
    np.fill_diagonal(trans, 0.0)
    cv = CarriedViterbi(trans, bound)
    total = 0
    for t0 in range(0, T, 10):
        labels, first, forced = cv.run(emis[t0:t0 + 10])
        assert first == total
        total += len(labels)
        assert cv.pending <= bound
    assert forced > 0
    labels, _, forced = cv.run(emis[:0], finish=True)
    assert total + len(labels) == T
