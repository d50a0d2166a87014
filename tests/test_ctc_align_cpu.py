"""CTC Viterbi with target and word timings, without a GPU: the NumPy contract (tests/ctc_align_reference.py) against
brute-force enumeration of every CTC path, on the tie rule and on infeasible / empty targets; the argument checks of
w2l_ctc_viterbi_target; and w2l_text_align_words (host code) on letters with `|`, surround + replabels (ASG), and
`_` word pieces (CTC), parsed by the field positions the `.align` consumers read."""
import ctypes
import itertools

import numpy as np
import pytest

import ctc_align_reference as R

LETTERS = "|\n'\n" + "\n".join("abcdefghijklmnopqrstuvwxyz") + "\n"


def brute_force(e, y):
    """every frame path over N tokens whose CTC collapse is y: (best float64 score, [paths at that score])"""
    T, N = e.shape
    best, arg = -np.inf, []
    for seq in itertools.product(range(N), repeat=T):
        if R.collapse(seq, N - 1) != list(y):
            continue
        sc = float(np.sum(e[np.arange(T), list(seq)], dtype=np.float64))
        if sc > best + 1e-9:
            best, arg = sc, [seq]
        elif abs(sc - best) <= 1e-9:
            arg.append(seq)
    return best, arg


def test_reference_is_the_best_path_by_enumeration():
    rng = np.random.default_rng(0)
    checked = unique = 0
    for T in range(1, 7):
        for N in range(2, 5):
            for L in range(0, 4):
                for _ in range(3):
                    e = rng.normal(0, 2, (1, T, N)).astype(np.float32)
                    y = rng.integers(0, N - 1, L).astype(np.int32)
                    tgt = np.full((1, 4), -1, np.int32)
                    tgt[0, :L] = y
                    path, state, score = R.ctc_viterbi_target(e, tgt, return_score=True)
                    best, arg = brute_force(e[0].astype(np.float64), y)
                    if not arg:  # no path spells y in T frames
                        assert (path == -1).all() and (state == -1).all() and L + np.sum(y[1:] == y[:-1]) > T
                        continue
                    checked += 1
                    got = float(np.sum(e[0, np.arange(T), path[0]], dtype=np.float64))
                    assert got == pytest.approx(best, abs=1e-5) and float(score[0]) == pytest.approx(best, abs=1e-4)
                    assert R.collapse(path[0], N - 1) == list(y)
                    if len(arg) == 1:
                        unique += 1
                        assert tuple(path[0]) == arg[0]
                    # the state path is a CTC path: starts in state 0 or 1, moves by 0, 1 or 2, ends in S-1 or S-2
                    S = 2 * L + 1
                    st = state[0]
                    assert st[0] in (0, 1) and st[-1] in (S - 1, S - 2) and set(np.diff(st)) <= {0, 1, 2}
                    assert all(path[0, t] == (N - 1 if st[t] % 2 == 0 else y[st[t] // 2]) for t in range(T))
    assert checked > 100 and unique > 50


def test_tie_rule_with_integer_emissions():
    # all-zero emissions: every path scores 0, the rule alone picks one
    # target [a], T=3: end state S-1 = 2 (alpha[1] == alpha[2]); back from (t=2, s=2): stay (tie with s-1)
    # -> (t=1, s=2): alpha_0[2] = -inf, alpha_0[1] = 0 -> s = 1
    p, s = R.ctc_viterbi_target(np.zeros((1, 3, 3), np.float32), np.array([[0]], np.int32))
    assert s.tolist() == [[1, 2, 2]] and p.tolist() == [[0, 2, 2]]
    # target [a, b], T=4: end 4; (3,4) stays; (2,4): alpha_1[4] = -inf -> 3; (1,3): alpha_0[3], alpha_0[2] = -inf,
    # skip from 1 allowed (b != a) -> 1
    p, s = R.ctc_viterbi_target(np.zeros((1, 4, 3), np.float32), np.array([[0, 1]], np.int32))
    assert s.tolist() == [[1, 3, 4, 4]] and p.tolist() == [[0, 1, 2, 2]]
    # a strictly greater later predecessor wins: label a scores 1 at frame 2.  End 2 (alpha_3[1] == alpha_3[2] = 1);
    # (3,2): alpha_2[1] = 1 > alpha_2[2] = 0 -> 1; (2,1) and (1,1): alpha[1] == alpha[0] = 0 -> stay
    e = np.zeros((1, 4, 3), np.float32)
    e[0, 2, 0] = 1.0
    p, s = R.ctc_viterbi_target(e, np.array([[0]], np.int32))
    assert s.tolist() == [[1, 1, 1, 2]] and p.tolist() == [[0, 0, 0, 2]]
    # end state S-2 only when strictly greater than S-1
    e = np.zeros((1, 2, 3), np.float32)
    e[0, 1, 0] = 1.0
    p, s = R.ctc_viterbi_target(e, np.array([[0]], np.int32))
    assert s.tolist() == [[1, 1]]


def test_empty_infeasible_and_invalid_targets():
    rng = np.random.default_rng(1)
    e = rng.normal(0, 1, (5, 4, 6)).astype(np.float32)
    tgt = np.array([[-1, -1, -1, -1, -1],      # empty: all blanks, state 0
                    [1, 1, 1, -1, -1],         # 3 labels + 2 repeats = 5 frames > 4: no alignment
                    [1, 2, 3, 4, 0],           # 5 labels > 4 frames
                    [1, -1, 2, -1, -1],        # a pad value inside the target: a label outside [0, N-1)
                    [1, 5, -1, -1, -1]],       # the blank as a label
                   np.int32)
    p, s = R.ctc_viterbi_target(e, tgt)
    assert p[0].tolist() == [5] * 4 and s[0].tolist() == [0] * 4
    for b in range(1, 5):
        assert (p[b] == -1).all() and (s[b] == -1).all()
    # exactly enough frames: the path is forced
    p, s = R.ctc_viterbi_target(e[:1], np.array([[2, 2, 3]], np.int32))
    assert s[0].tolist() == [1, 2, 3, 5] and p[0].tolist() == [2, 5, 2, 3]


def test_abi_argument_errors():
    from wav2letter_b200 import capi

    lib = capi.lib
    one = ctypes.c_void_p(256)  # never dereferenced: validation fails first
    assert lib.w2l_ctc_viterbi_workspace_size(16, 1500, 10000, 500) >= 16 * 1500 * 1024 * 4 + 16 * 1500 * 64 * 4
    assert lib.w2l_ctc_viterbi_workspace_size(0, 10, 30, 5) == 0
    assert lib.w2l_ctc_viterbi_target(None, 0, 10, 30, 5, one, one, one, None, one, 1 << 30) == 1
    assert lib.w2l_ctc_viterbi_target(None, 2, 10, 1, 5, one, one, one, None, one, 1 << 30) == 1
    assert lib.w2l_ctc_viterbi_target(None, 2, 10, 30, 5, None, one, one, None, one, 1 << 30) == 1
    assert lib.w2l_ctc_viterbi_target(None, 2, 10, 30, 5, one, None, one, None, one, 1 << 30) == 1
    assert lib.w2l_ctc_viterbi_target(None, 2, 2000, 30, 1024, one, one, one, None, one, 1 << 40) == 4
    assert lib.w2l_ctc_viterbi_target(None, 2, 10, 30, 5, one, one, one, None, one, 16) == 2
    assert b"workspace" in lib.w2l_last_error()


def frames(*runs):
    """idx per frame from (index, repeat) runs"""
    return np.concatenate([np.full(n, i, np.int32) for i, n in runs])


def parse(line):
    """the fields the in-tree consumers read: id TAB segments joined by a literal backslash-n; per segment, field 2 is
    the begin time, field 3 the duration, field 4 the word"""
    utt, rest = line.split("\t")
    segs = []
    for seg in rest.strip().split("\\n"):
        f = seg.split()
        assert len(f) == 5 and f[0] == utt and f[1] == "1"
        segs.append((float(f[2]), float(f[3]), f[4]))
    return utt, segs


def check_tiling(segs, total_s):
    assert segs[0][2] == "$" and segs[0][0] == 0.0  # the consumers skip the first segment
    for (b0, d0, _), (b1, _, _) in zip(segs, segs[1:]):
        assert b1 == pytest.approx(b0 + d0, abs=1e-6)
    assert segs[-1][0] + segs[-1][1] == pytest.approx(total_s, abs=1e-6)


def test_word_timings_ctc_letters():
    from wav2letter_b200.text import TextPipeline

    tp = TextPipeline(LETTERS, "", "ctc", 0, "", False, "|")
    tgt = tp.encode("hello hi")  # h e l l o | h i |
    assert len(tgt) == 9
    # blank x3, h x2, e x2, l, blank (between the two l), l x2, o, | x3, h, blank x2, i x2, |, blank x2
    idx = frames((0, 3), (1, 2), (3, 2), (5, 1), (6, 1), (7, 2), (9, 1), (11, 3), (13, 1), (14, 2), (15, 2), (17, 1), (18, 2))
    line = tp.align_words(np.concatenate([tgt, [-1, -1]]), idx, 80.0, "utt-1")
    utt, segs = parse(line)
    assert utt == "utt-1"
    assert segs == [(0.0, 0.24, "$"), (0.24, 0.72, "hello"), (0.96, 0.24, "$"), (1.2, 0.4, "hi"), (1.6, 0.24, "$")]
    check_tiling(segs, 23 * 0.08)


def test_word_timings_asg_surround_and_replabels():
    from wav2letter_b200.text import TextPipeline

    tp = TextPipeline(LETTERS, "", "asg", 2, "|", False, "|")
    tgt = tp.encode("hello all")  # | h e l <1> o | a l <1> | <1>
    assert len(tgt) == 12
    idx = frames((0, 2), (1, 1), (2, 1), (3, 2), (4, 1), (5, 1), (6, 3), (7, 1), (8, 1), (9, 1), (10, 2), (11, 1))
    _, segs = parse(tp.align_words(tgt, idx, 40.0, "a"))
    assert [w for _, _, w in segs] == ["$", "hello", "$", "all", "$"]
    assert segs[1] == (0.08, 0.24, "hello") and segs[3] == (0.44, 0.12, "all")
    check_tiling(segs, 17 * 0.04)


def test_word_timings_ctc_word_pieces():
    from wav2letter_b200.text import TextPipeline

    tp = TextPipeline("_he\nllo\n_wor\nld\n", "hello _he llo\nworld _wor ld\n", "ctc", 0, "", True, "_")
    tgt = tp.encode("hello world")
    assert tgt.tolist() == [0, 1, 2, 3]
    idx = frames((1, 2), (3, 1), (4, 2), (5, 1), (7, 1), (8, 1))  # the blank between the words is silence
    _, segs = parse(tp.align_words(tgt, idx, 10.0, "wp"))
    assert segs == [(0.0, 0.0, "$"), (0.0, 0.03, "hello"), (0.03, 0.02, "$"), (0.05, 0.02, "world"), (0.07, 0.01, "$")]


def test_word_timings_reject_partial_alignments():
    from wav2letter_b200 import W2LError
    from wav2letter_b200.text import TextPipeline

    tp = TextPipeline(LETTERS, "", "ctc", 0, "", False, "|")
    tgt = tp.encode("ab")
    with pytest.raises(W2LError):
        tp.align_words(tgt, np.full(5, -1, np.int32), 10.0, "x")  # no alignment
    with pytest.raises(W2LError):
        tp.align_words(tgt, frames((1, 2), (3, 2)), 10.0, "x")  # stops before the last label
    asg = TextPipeline(LETTERS, "", "asg", 0, "", False, "|")
    with pytest.raises(W2LError):
        asg.align_words(asg.encode("ab"), frames((0, 2), (1, 2)), 10.0, "x")
