"""slimIPL without a GPU: the float64 soft-label loss model against torch float64 autograd, the float32 EMA model's
rounding, and the hard pseudo-label text round trip of Train.cpp:1376-1407 (path -> letters -> words -> " ".join ->
targets) on hand-made paths."""
import numpy as np
import pytest
import torch

import slimipl_reference as ref

LETTERS = "|\n'\n" + "\n".join("abcdefghijklmnopqrstuvwxyz") + "\n"


def idx(ch):
    return {"|": 0, "'": 1}.get(ch, 2 + ord(ch) - ord("a") if ch.isalpha() else None)


@pytest.mark.parametrize("shape,scale,peak", [((1, 29), 1.0, 1.0), ((3, 5, 17), 0.5, 1.0), ((2, 7, 100), 2.0, 50.0)])
def test_soft_loss_model_matches_torch_autograd(shape, scale, peak):
    rng = np.random.default_rng(sum(shape))
    z = rng.standard_normal(shape) * 3
    t = rng.standard_normal(shape) * peak
    loss, d = ref.soft_label_loss(z, t, scale)
    zt = torch.tensor(z, dtype=torch.float64, requires_grad=True)
    tt = torch.tensor(t, dtype=torch.float64)
    # Train.cpp:1666-1673: softScale * -mean_{frames, utterances} sum_c softmax(teacher) * logSoftmax(student)
    want = scale * -(torch.softmax(tt, -1) * torch.log_softmax(zt, -1)).sum(-1).mean()
    want.backward()
    want = float(want.detach())
    assert abs(loss - want) <= 1e-12 * max(1.0, abs(want))
    np.testing.assert_allclose(d, zt.grad.numpy(), rtol=1e-10, atol=1e-15)


def test_soft_loss_model_of_identical_rows_has_zero_gradient_and_the_entropy():
    rng = np.random.default_rng(3)
    z = rng.standard_normal((4, 33))
    loss, d = ref.soft_label_loss(z, z, 1.0)
    assert np.abs(d).max() < 1e-15
    p = np.exp(z) / np.exp(z).sum(-1, keepdims=True)
    assert abs(loss - float(-(p * np.log(p)).sum(-1).mean())) < 1e-12


@pytest.mark.parametrize("decay", [0.0, 0.5, 0.9, 0.999, 1.0, 1.0 / 3.0])
def test_ema_model_rounds_each_product_and_the_sum_once(decay):
    rng = np.random.default_rng(int(decay * 1000))
    e = rng.standard_normal(4096).astype(np.float32)
    p = rng.standard_normal(4096).astype(np.float32)
    got = ref.ema_update(e, p, decay)
    assert got.dtype == np.float32
    d, omd = np.float32(decay), np.float32(1.0 - decay)
    # a product of two float32 is exact in float64: rounding it to float32 is the correctly rounded float32 product
    a = (e.astype(np.float64) * np.float64(d)).astype(np.float32)
    b = (p.astype(np.float64) * np.float64(omd)).astype(np.float32)
    want = (a.astype(np.float64) + b.astype(np.float64)).astype(np.float32)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    if decay == 0.0:
        assert np.array_equal(got, p)
    if decay == 1.0:
        assert np.array_equal(got, e)


def _text(criterion="ctc", replabel=0, lexicon="", tokens=LETTERS):
    from wav2letter_b200.text import TextPipeline

    return TextPipeline(tokens, lexicon, criterion, replabel, "", False, "|")


def _round_trip(tp, paths):
    from wav2letter_b200.slimipl import pl_strings

    strings = pl_strings(tp, paths)
    return strings, tp.encode_batch(strings)


def test_pl_round_trip_collapses_repeats_and_drops_blanks():
    tp = _text("ctc")
    blank = tp.num_classes - 1
    path = [blank, idx("h"), idx("h"), idx("i"), blank, blank, idx("y"), idx("o"), idx("o"), blank]
    strings, tgt = _round_trip(tp, [path])
    assert strings == ["hiyo"]
    assert tgt[0].tolist() == tp.encode("hiyo").tolist()
    # a blank between equal letters keeps both
    strings, _ = _round_trip(tp, [[idx("a"), blank, idx("a"), idx("b")]])
    assert strings == ["aab"]


def test_pl_round_trip_separators_around_a_blank_make_one_word_break():
    tp = _text("ctc")
    blank = tp.num_classes - 1
    sep = idx("|")
    paths = np.array([[idx("h"), idx("i"), sep, blank, sep, idx("y"), idx("o"), sep, sep],
                      [sep, idx("a"), blank, blank, blank, blank, blank, blank, blank]], np.int32)
    strings, tgt = _round_trip(tp, paths)
    assert strings == ["hi yo", "a"]
    assert tgt.shape == (2, len(tp.encode("hi yo")))
    assert tgt[0].tolist() == tp.encode("hi yo").tolist()
    assert tgt[1].tolist()[:2] == tp.encode("a").tolist() and set(tgt[1].tolist()[2:]) == {-1}


def test_pl_round_trip_unknown_word_falls_back_to_letters():
    tp = _text("ctc", lexicon="hi h i |\n")
    blank = tp.num_classes - 1
    path = [idx("h"), idx("i"), idx("|"), blank, idx("z"), blank, idx("z"), idx("|")]
    strings, tgt = _round_trip(tp, [path])
    assert strings == ["hi zz"]
    assert tgt[0].tolist() == [idx("h"), idx("i"), idx("|"), idx("z"), idx("z"), idx("|")]


def test_pl_round_trip_seq2seq_cuts_at_eos():
    tp = _text("seq2seq", tokens="|\na\nb\nc\n")
    eos, pad = 4, 5
    path = [1, 2, 0, 3, eos, 1, 1, pad]  # "ab c", then eos; what follows it is not part of the PL
    strings, tgt = _round_trip(tp, [path, [3, eos, 2, 2, 2, 2, 2, 2]])
    assert strings == ["ab c", "c"]
    assert tgt[0].tolist() == [1, 2, 0, 3, 0, eos]
    assert tgt[1].tolist() == [3, 0, eos, pad, pad, pad]


def test_pl_round_trip_replabel_2():
    tp = _text("asg", replabel=2)
    R1, R2 = 28, 29
    # ASG Viterbi paths stay several frames on a token: "a <2>" spells "aaa", "l <1>" spells "ll"
    path = np.repeat([idx("a"), R2, idx("|"), idx("b"), idx("e"), idx("l"), R1, idx("|")], 3)
    strings, tgt = _round_trip(tp, [path])
    assert strings == ["aaa bell"]
    assert tgt[0].tolist() == tp.encode("aaa bell").tolist()
    assert tgt[0].tolist() == [idx("a"), R2, idx("|"), idx("b"), idx("e"), idx("l"), R1, idx("|")]


@pytest.mark.parametrize("version,known", [(3, False), (4, True), (5, False)])
def test_checkpoint_versions_around_the_teacher_format(tmp_path, version, known):
    """version 4 (a trainer with a teacher) is read; version 3 stays unknown, as does anything past 4"""
    import struct

    from wav2letter_b200 import capi

    p = tmp_path / "ck.bin"
    p.write_bytes(b"W2LB200\0" + struct.pack("<I", version) + b"\0" * 64)
    assert not capi.lib.w2l_trainer_load(None, str(p).encode())
    assert (b"unsupported version" not in capi.lib.w2l_last_error()) == known
