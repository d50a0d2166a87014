"""The model of the device scoring contract (tests/eval_reference.py) against the host pipeline it stands for:
prediction2ltr / target2ltr / ltr2wrd / EditDistanceMeter (host/text_pipeline.cpp), on random rows for every setting
the recipes combine: criterion ctc / asg / seq2seq, replabel 0 / 2, surround none / "|", word pieces off / on, with
multi-byte UTF-8 tokens."""
import itertools
import random
import zlib

import pytest

import eval_reference as ref

GRID = list(itertools.product(["ctc", "asg", "seq2seq"], [0, 2], ["", "|"], [False, True]))


def host_counts(tp, path, target):
    from wav2letter_b200 import W2LError
    from wav2letter_b200.text import EditDistanceMeter

    try:
        hl, rl = tp.prediction2ltr(path), tp.target2ltr(target)
        hw, rw = tp.ltr2wrd(hl), tp.ltr2wrd(rl)
    except W2LError:
        return [-1] * 8
    ml, mw = EditDistanceMeter(), EditDistanceMeter()
    ml.add(hl, rl)
    mw.add(hw, rw)
    return list(ml.raw()) + list(mw.raw())


def make(args):
    from wav2letter_b200.text import TextPipeline

    return TextPipeline("\n".join(args["tokens"]) + "\n", "", args["criterion"], args["replabel"], args["surround"], args["wordpiece"],
                        args["wordsep"])


@pytest.mark.parametrize("criterion,replabel,surround,wordpiece", GRID)
def test_model_matches_host(criterion, replabel, surround, wordpiece):
    args = ref.pipeline_args(criterion, replabel, surround, wordpiece)
    tp, t = make(args), ref.Tables(**args)
    assert t.N == tp.num_classes
    rng = random.Random(zlib.crc32(repr((criterion, replabel, surround, wordpiece)).encode()))
    rejected = 0
    for _ in range(400):
        path = ref.random_row(rng, t, rng.randrange(0, 40), True)
        target = ref.random_row(rng, t, rng.randrange(1, 25), False, invalid_rate=0.002, minus_one=0.005)
        want = host_counts(tp, path, target)
        assert ref.counts(t, path, target) == want, (path, target)
        rejected += want[0] < 0
    assert 0 < rejected < 100  # most cases are scored, some refused


def test_tie_order_and_word_bytes():
    t = ref.Tables(ref.LETTER_TOKENS, "asg")
    a, b, ab, sep = (ref.LETTER_TOKENS.index(c) for c in ("a", "b", "ab", "|"))
    # "ab" against "ba": the total is 2 whichever way, the preference order makes it two substitutions
    assert ref.edit([1, 2], [2, 1]) == (0, 0, 2)
    assert ref.counts(t, [a, b], [b, a])[:4] == [2, 0, 0, 2]
    # the token "ab" and the letters a, b spell the same word: one letter apart, equal as words
    c = ref.counts(t, [ab, sep, a], [a, b, sep, a])
    assert c[4:] == [2, 0, 0, 0] and c[:4] == [4, 1, 0, 1]
