"""CPU checks of the Seq2Seq criterion's float64 oracle (oracle/seq2seq_ref.py), the NumPy model of its token
substitution (tests/seq2seq_reference.py) and the seq2seq text pipeline."""
import math

import numpy as np
import torch

import seq2seq_reference as S
from oracle import seq2seq_ref as ref


def test_window_closed_form():
    w = ref.window(4, 10, 2.0)
    assert w.shape == (4, 10)
    for u in range(4):
        for t in range(10):
            c = u * 10 / 4
            assert math.isclose(float(w[u, t]), -((t - c) ** 2) / 8.0, rel_tol=0, abs_tol=1e-12)
    assert float(w[2, 5]) == 0.0  # the window's centre for u = 2 is t = 5


def test_attention_with_window_is_softmax_of_shifted_scores():
    g = torch.Generator().manual_seed(0)
    q = torch.randn(1, 3, 4, dtype=torch.float64, generator=g)
    x = torch.randn(1, 6, 8, dtype=torch.float64, generator=g)
    win = ref.window(3, 6, 1.5)
    got = ref.attention(q, x, win)
    for u in range(3):
        s = [float(q[0, u] @ x[0, t, :4]) / 2.0 + float(win[u, t]) for t in range(6)]
        a = np.exp(np.array(s) - max(s))
        a /= a.sum()
        want = q[0, u].numpy() + (a[:, None] * x[0, :, 4:].numpy()).sum(0)
        np.testing.assert_allclose(got[0, u].numpy(), want, rtol=1e-12, atol=1e-12)


def small_model(N=7, H=4, R=1, L=1, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(*s, dtype=torch.float64, generator=g) * 0.5).requires_grad_(True) for s in ref.param_shapes(N, H, R, L)]


def test_label_smoothing_closed_form():
    N, H, B, T, U = 7, 4, 2, 5, 4
    params = small_model(N, H)
    x = torch.randn(B, T, 2 * H, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    y = np.array([[1, 2, 5, 6], [3, 5, 6, 6]])  # eos = 5, pad = 6
    tok = ref.teacher_tokens(y, N)
    lp = torch.log_softmax(ref.logits(params, x, tok), -1)
    for ls in (0.0, 0.05):
        got = ref.loss(params, x, y, 6, tok, labelsmooth=ls)
        for b in range(B):
            want = 0.0
            for u in range(U):
                if y[b, u] == 6:
                    continue
                want += -(1 - ls) * float(lp[b, u, y[b, u]].detach()) - ls / N * float(lp[b, u].sum().detach())
            assert math.isclose(float(got[b]), want, rel_tol=1e-12)


def test_pad_rows_contribute_nothing():
    N, H, B, T = 7, 4, 1, 5
    params = small_model(N, H)
    x = torch.randn(B, T, 2 * H, dtype=torch.float64, generator=torch.Generator().manual_seed(2))
    short = np.array([[1, 2, 5]])
    long = np.array([[1, 2, 5, 6, 6, 6]])
    a = ref.loss(params, x, short, 6, ref.teacher_tokens(short, N))
    b = ref.loss(params, x, long, 6, ref.teacher_tokens(long, N))
    assert math.isclose(float(a), float(b), rel_tol=1e-12)
    b.sum().backward()
    gb = [p.grad.clone() for p in params]
    for p in params:
        p.grad = None
    a.sum().backward()
    for p, q in zip(params, gb):
        torch.testing.assert_close(p.grad, q, rtol=1e-12, atol=1e-14)


def test_substitution_rate():
    y = np.tile(np.arange(40) % 11, (64, 1))
    assert (S.substituted_tokens(0x5EED0000, y, 13, 100) == ref.teacher_tokens(y, 13).numpy()).all()
    for pct in (99, 80, 50):
        tok = S.substituted_tokens(0x1234567890ABCDEF, y, 13, pct)
        assert (tok[:, 0] == 13).all()
        assert tok[:, 1:].max() <= 11 and tok[:, 1:].min() >= 0
        # a replacement may draw the original token: the changed fraction is q (N - 2) / (N - 1) on average
        q = 1 - pct / 100
        changed = (tok[:, 1:] != y[:, :-1]).mean()
        expect = q * 11 / 12
        n = y[:, 1:].size
        assert abs(changed - expect) < 5 * math.sqrt(expect * (1 - expect) / n) + 1e-3, (pct, changed, expect)


def test_text_pipeline_seq2seq():
    from wav2letter_b200.text import TextPipeline

    tokens = "|\na\nb\nc\n"
    tp = TextPipeline(tokens, criterion="seq2seq", wordsep="|")
    assert tp.num_classes == 6  # | a b c, then eos, then pad
    eos, pad = 4, 5
    assert tp.pad_index == pad
    enc = tp.encode("ab c")
    assert list(enc) == [1, 2, 0, 3, 0, eos]  # letter fallback, word separator on the right, then eos
    batch = tp.encode_batch(["ab c", "a"])
    assert batch.shape == (2, 6) and list(batch[1]) == [1, 0, eos, pad, pad, pad]
    assert tp.prediction2ltr([1, 2, 0, 3, eos, 1, 1, pad]) == ["a", "b", "|", "c"]
    assert tp.prediction2ltr([1, 1, pad, pad]) == ["a", "a"]
    assert tp.target2ltr(batch[1]) == ["a"]
    ctc = TextPipeline(tokens, criterion="ctc", wordsep="|")
    assert ctc.num_classes == 5 and ctc.pad_index == -1
