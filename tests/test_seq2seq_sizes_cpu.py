"""CPU checks of the Seq2Seq criterion on padded batches: the frame-count rule, the sized float64 reference against the
unsized oracle and against each utterance run on its own frames, and the argument checks of the new entry points that
fail before anything is launched."""
import ctypes

import numpy as np
import pytest
import torch

import seq2seq_sizes_reference as SR
from oracle import seq2seq_ref as ref


def test_frame_counts():
    assert SR.frame_counts([1200, 1199, 1000, 7], 150)[0] == [150, 150, 125, 1]
    assert SR.frame_counts([640], 150)[0] == [150]  # one utterance alone masks nothing
    assert SR.frame_counts([10, 9, 1], 4)[0] == [4, 4, 1]  # ceil(3.6) = 4, ceil(0.4) = 1
    assert SR.frame_counts([100.0, 50.0], 7)[0] == [7, 4]  # whole-number floats; ceil(3.5) = 4
    tps, ups, bad = SR.frame_counts([100, 0, -3, 50], 10, [5, 1, 6, 0], 5)
    assert tps == [10, 10, 10, 5] and ups == [5, 1, 5, 5] and bad == [False, True, True, True]
    assert SR.frame_counts([0, -1], 10)[2] == [True, True]  # no positive duration
    assert SR.frame_counts([10.5, 10.0], 10)[2] == [True, False]


def params(N, H, R, L, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.rand(s, generator=g, dtype=torch.float64) - 0.5).requires_grad_(True) for s in ref.param_shapes(N, H, R, L)]


def batch(B, Tp, U, H, N, seed):
    rng = np.random.default_rng(seed)
    x = torch.from_numpy(rng.standard_normal((B, Tp, 2 * H))).requires_grad_(True)
    y = np.full((B, U), N - 1, np.int64)
    for b in range(B):
        n = int(rng.integers(1, U))
        y[b, :n] = rng.integers(0, N - 2, n)
        y[b, n] = N - 2
    return x, y


@pytest.mark.parametrize("window_std", [0.0, 3.0])
def test_full_sizes_equal_the_oracle(window_std):
    N, H, B, Tp, U, R, L = 11, 8, 3, 12, 6, 2, 2
    p = params(N, H, R, L, 1)
    x, y = batch(B, Tp, U, H, N, 2)
    tok = ref.teacher_tokens(y, N)
    want = ref.loss(p, x, y, N - 1, tok, R, L, window_std, 0.1)
    gw = torch.autograd.grad(want.sum(), [x] + p)
    got = SR.loss(p, x, y, N - 1, tok, [Tp] * B, [U] * B, R, L, window_std, 0.1)
    gg = torch.autograd.grad(got.sum(), [x] + p)
    assert torch.equal(got, want)
    for a, b in zip(gg, gw):
        assert torch.equal(a, b)


@pytest.mark.parametrize("window_std", [0.0, 3.0])
def test_padded_batch_is_each_utterance_alone(window_std):
    """loss and encoder gradient of a padded batch with NaN padding = the oracle on x[b, :T'_b] and y[b, :U_b]"""
    N, H, B, Tp, U, R, L = 11, 8, 3, 12, 7, 1, 2
    p = params(N, H, R, L, 3)
    x, y = batch(B, Tp, U, H, N, 4)
    tps, _, _ = SR.frame_counts([120, 61, 30], Tp)
    ups = [int(np.argmax(y[b] == N - 2)) + 1 for b in range(B)]
    with torch.no_grad():
        for b in range(B):
            x[b, tps[b]:] = float("nan")
    got = SR.loss(p, x, y, N - 1, ref.teacher_tokens(y, N), tps, ups, R, L, window_std)
    (dx,) = torch.autograd.grad(got.sum(), [x])
    for b in range(B):
        xb = x[b:b + 1, :tps[b]].detach().clone().requires_grad_(True)
        yb = y[b:b + 1, :ups[b]]
        want = ref.loss(p, xb, yb, N - 1, ref.teacher_tokens(yb, N), R, L, window_std)
        (dxb,) = torch.autograd.grad(want.sum(), [xb])
        assert abs(float((got[b] - want[0]).detach())) <= 1e-12 * max(1.0, abs(float(want[0].detach())))
        assert torch.allclose(dx[b, :tps[b]], dxb[0], rtol=1e-10, atol=1e-12)
        assert (dx[b, tps[b]:] == 0).all()


def test_sized_greedy_is_each_utterance_alone():
    N, H, B, Tp, R, L, maxlen = 11, 8, 4, 12, 2, 1, 9
    p = params(N, H, R, L, 5)
    x, _ = batch(B, Tp, 3, H, N, 6)
    tps = [12, 5, 1, 9]
    with torch.no_grad():
        xp = x.detach().clone()
        for b in range(B):
            xp[b, tps[b]:] = float("nan")
        got = SR.greedy(p, xp, tps, N - 2, maxlen, R, L)
        for b in range(B):
            want = ref.greedy(p, x.detach()[b:b + 1, :tps[b]], N - 2, maxlen, R, L)[0]
            assert got[b][0] == want[0]
            assert np.allclose(got[b][1], want[1], rtol=1e-10, atol=1e-12)


def test_argument_checks_before_any_launch():
    from wav2letter_b200 import capi
    from wav2letter_b200.trainer import size_arg

    lib = capi.lib
    one = ctypes.c_void_p(256)  # never dereferenced: validation fails first
    assert lib.w2l_seq2seq_sizes(None, 0, 10, 5, one, 0, one, one, one, None) == 1
    assert lib.w2l_seq2seq_sizes(None, 2, 10, 5, one, 2, one, one, one, None) == 1
    assert lib.w2l_seq2seq_sizes(None, 2, 10, 5, one, 0, one, None, one, None) == 1
    assert lib.w2l_seq2seq_attn_fwd_sized(None, 2, 3, 10, 48, one, one, one, one, 3, 0.0, one, None) == 4  # H % 32
    assert lib.w2l_seq2seq_attn_fwd_sized(None, 2, 3, 10, 32, None, one, one, one, 3, 0.0, one, None) == 1
    assert lib.w2l_seq2seq_attn_bwd_sized(None, 2, 3, 10, 32, one, one, one, one, one, one, None, one) == 1
    assert size_arg(None, 3, "input_sizes") is None
    with pytest.raises(ValueError, match="2 entries for a batch of 3"):
        size_arg([1, 2], 3, "input_sizes")
    with pytest.raises(TypeError):
        size_arg([1.5, 2, 3], 3, "input_sizes")
    with pytest.raises(TypeError):
        size_arg(torch.ones(3, dtype=torch.int32), 3, "input_sizes")  # not on the GPU
    with pytest.raises(ValueError, match="int32"):
        size_arg([1, 2, 1 << 40], 3, "target_sizes")
