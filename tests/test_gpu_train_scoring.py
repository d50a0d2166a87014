"""Scored training steps (Trainer.step(..., text=...), w2l_trainer_step_scored; DESIGN.md §10): Train.cpp's train meters
(:1699-1714) from the step's own training-mode output.

- the CTC argmax fused into the loss's prep pass (w2l_ctc_forward_backward_path) equals w2l_argmax_path bit for bit, and
  the loss and gradient are those of the call without it;
- scoring does not perturb training: losses and parameter arenas of k scored steps equal those of k unscored steps;
- the counts are the step's own: where the training-mode forward equals the eval-mode one they equal the host pipeline's
  rows of viterbi_path, and an overfitted model scores no training errors;
- a mixed-precision step that retries returns the counts of the same batch at the final scale;
- refusals leave parameters, position and loss scaling untouched."""
import numpy as np
import pytest
import torch

import test_gpu_slimipl as sl
from test_gpu_eval import _host_rows

pytestmark = pytest.mark.gpu

# TDS_ARCH with SpecAugment and dropout: its training-mode forward differs from the eval-mode one
DROP_ARCH = """V -1 NFEAT 1 0
SAUG 0 4 2 10 1.0 2
C2 1 4 5 1 1 1 -1 -1
R
DO 0.2
TDS 4 5 16 0.2
V 0 64 1 0
RO 1 0 3 2
L 64 NLABEL
"""


def _bits(x):
    return x.contiguous().view(torch.int32)


# ---- the fused argmax --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [2, 30, 32, 33, 10000])
def test_fused_argmax_equals_argmax_path(N):
    from wav2letter_b200 import argmax_path, ctc_forward_backward

    B, T, L = 3, 7, 4  # B T = 21 frames: not a multiple of the 8 warps of a CTA
    g = torch.Generator(device="cuda").manual_seed(N)
    e = torch.randn((B, T, N), device="cuda", generator=g)
    e[0, 0] = 1.5                                    # every element ties
    if N > 35:
        e[0, 1, 3] = e[0, 1, 35] = e[0, 1].max() + 1  # a tie between lanes 3 (index 3) and 3 (index 35)
        e[0, 2, 34] = e[0, 2, 1] = e[0, 2].max() + 1  # lanes 2 and 1: the lower index wins
    e[1, 0] = float("-inf")                          # all -inf
    e[1, 1, 0] = float("nan")                        # NaN seeds lane 0
    e[1, 2, N - 1] = float("nan")                    # NaN later in a row
    e[1, 3] = float("nan")                           # all NaN
    tgt = torch.randint(0, N - 1, (B, L), device="cuda", generator=g, dtype=torch.int32)
    want = argmax_path(e)
    dloss = torch.rand(B, device="cuda", generator=g) + 0.5
    for need_grad in (False, True):
        l0, d0 = ctc_forward_backward(e, tgt, "target_sz", dloss=dloss, need_grad=need_grad)
        path = torch.full((B, T), -7, dtype=torch.int32, device="cuda")
        l1, d1 = ctc_forward_backward(e, tgt, "target_sz", dloss=dloss, need_grad=need_grad, path=path)
        assert torch.equal(path, want), (need_grad, path, want)
        assert torch.equal(_bits(l0), _bits(l1))
        if need_grad:
            assert torch.equal(_bits(d0), _bits(d1))
    # the clean utterance: a finite loss and the argmax of every frame
    assert torch.isfinite(l0[2]) and torch.equal(want[2].long(), e[2].argmax(-1))


def test_ctc_needs_two_classes():
    from wav2letter_b200 import W2LError, ctc_forward_backward

    e = torch.zeros((1, 4, 1), device="cuda")
    with pytest.raises(W2LError):
        ctc_forward_backward(e, torch.zeros((1, 1), dtype=torch.int32, device="cuda"),
                             path=torch.zeros((1, 4), dtype=torch.int32, device="cuda"))


# ---- the trainer -------------------------------------------------------------------------------------------------------
def _text(criterion):
    from wav2letter_b200.text import TextPipeline

    c = "ctc" if criterion == "ctc" else "asg"
    return TextPipeline(sl.LETTERS, "", c, 0 if c == "ctc" else 2, "" if c == "ctc" else "|", False, "|")


def _seeded_trainer(criterion, arch, N, precision, seed):
    from wav2letter_b200.capi import lib

    lib.w2l_set_seed(seed)
    return sl._trainer(criterion, N=N, lr=0.05, momentum=0.9, precision=precision, arch=arch, maxgradnorm=1.0)


@pytest.mark.parametrize("criterion", ["ctc", "asg", "linseg"])
@pytest.mark.parametrize("precision", ["f32", "bf16"])
@pytest.mark.parametrize("grad_stream", [True, False])
def test_scoring_does_not_perturb_training(criterion, precision, grad_stream):
    from wav2letter_b200.capi import lib

    text = _text(criterion)
    N = text.num_classes
    rng = np.random.default_rng(7)
    feat = sl._spoken(rng, text, sl.TRANSCRIPTS)
    tgt = torch.from_numpy(text.encode_batch(sl.TRANSCRIPTS)).cuda()
    runs = []
    for scored in (False, True):
        tr = _seeded_trainer(criterion, DROP_ARCH, N, precision, 1234)
        tr.set_grad_stream(grad_stream)
        lib.w2l_set_seed(99)
        losses, counts = [], []
        for _ in range(4):
            if scored:
                loss, c = tr.step(feat, tgt, text=text)
                counts.append(c.clone())
            else:
                loss = tr.step(feat, tgt)
            losses.append(loss.clone())
        runs.append((losses, tr.get_flat(0).clone(), tr.get_flat(1).clone(), counts))
        tr.close()
    (l0, p0, c0, _), (l1, p1, c1, counts) = runs
    for a, b in zip(l0, l1):
        assert torch.equal(_bits(a), _bits(b))
    assert torch.equal(_bits(p0), _bits(p1)) and torch.equal(_bits(c0), _bits(c1))
    # with dropout the paths differ from step to step, but the reference columns are the target's alone
    ref = _host_rows(text, torch.zeros((len(sl.TRANSCRIPTS), 1), dtype=torch.int32, device="cuda"), tgt)
    for c in counts:
        c = c.cpu().numpy()
        assert (c[:, 0] == ref[:, 0]).all() and (c[:, 4] == ref[:, 4]).all()


@pytest.mark.parametrize("criterion,arch", [("ctc", sl.TDS_ARCH), ("asg", None), ("linseg", None)])
def test_counts_are_the_steps_own(criterion, arch):
    """no dropout or SAUG: the step's output is the eval-mode output, so counts = scoring of viterbi_path just before"""
    import test_gpu_convglu as cg
    from wav2letter_b200.text import ErrorRates

    text = _text(criterion)
    tr = sl._trainer(criterion, N=text.num_classes, lr=0.05, momentum=0.9, arch=arch or cg.ARCH, maxgradnorm=1.0)
    rng = np.random.default_rng(3)
    feat = sl._spoken(rng, text, sl.TRANSCRIPTS)
    tgt = torch.from_numpy(text.encode_batch(sl.TRANSCRIPTS)).cuda()
    for i in range(20 if criterion == "linseg" else 3000):
        path = tr.viterbi_path(feat)
        want = text.edit_counts(path, tgt)
        _, counts = tr.step(feat, tgt, total_batch=3.0, text=text)
        assert torch.equal(counts, want), i
        if i % 50 == 0:
            assert np.array_equal(counts.cpu().numpy(), _host_rows(text, path, tgt))
        if criterion != "linseg" and (counts[:, 1:4].sum() + counts[:, 5:8].sum()).item() == 0:
            break
    if criterion != "linseg":  # (the linear-segmentation warm start is not trained to convergence)
        m = ErrorRates()
        m.add(counts)
        assert m.ter() == 0.0 and m.wer() == 0.0
    tr.close()


def test_retried_step_counts_equal_the_final_scale():
    """fp16 with a loss scale whose backward overflows: the step retries at half the scale on the same random draws, and
    its counts are those of the same batch run at the final scale without retries"""
    text = _text("ctc")
    N = text.num_classes
    rng = np.random.default_rng(11)
    feat = sl._spoken(rng, text, sl.TRANSCRIPTS)
    tgt = torch.from_numpy(text.encode_batch(sl.TRANSCRIPTS)).cuda()
    tr = _seeded_trainer("ctc", DROP_ARCH, N, "fp16", 77)
    p0 = tr.get_flat(0).clone()
    tr.set_amp(True, initial_scale=2.0 ** 40)
    from wav2letter_b200.capi import lib

    lib.w2l_set_seed(5)
    _, counts = tr.step(feat, tgt, text=text)
    retries = tr.amp_state()[2]
    assert retries > 0
    final = 2.0 ** 40 / 2.0 ** retries
    after = tr.get_flat(0).clone()
    tr.close()
    fresh = _seeded_trainer("ctc", DROP_ARCH, N, "fp16", 77)
    assert torch.equal(fresh.get_flat(0), p0)
    fresh.set_amp(True, initial_scale=final)
    lib.w2l_set_seed(5)
    _, c2 = fresh.step(feat, tgt, text=text)
    assert fresh.amp_state()[2] == 0
    assert torch.equal(counts, c2) and torch.equal(_bits(after), _bits(fresh.get_flat(0)))
    fresh.close()


def test_refusals_change_nothing():
    import test_gpu_seq2seq as s2s
    from wav2letter_b200 import W2LError
    from wav2letter_b200.capi import _ptr, _stream, lib

    text = _text("ctc")
    N = text.num_classes
    tr = sl._trainer("ctc", N=N, lr=0.05, momentum=0.9, maxgradnorm=1.0)
    tr.set_amp(True, initial_scale=64.0)
    rng = np.random.default_rng(4)
    feat = sl._spoken(rng, text, sl.TRANSCRIPTS)
    tgt = torch.from_numpy(text.encode_batch(sl.TRANSCRIPTS)).cuda()
    tr.step(feat, tgt, text=text)
    state = (tr.get_flat(0).clone(), tr.get_flat(1).clone(), tr.position(), tr.amp_state())
    B, T, L = feat.shape[0], feat.shape[3], tgt.shape[1]
    counts = torch.empty((B, 8), dtype=torch.int32, device="cuda")
    loss = torch.empty(B, device="cuda")
    dev = text.to_device()
    wide = torch.full((B, (1 << 20) + 1), -1, dtype=torch.int32, device="cuda")  # beyond the scorer's target width
    calls = {
        "asg text": lambda: lib.w2l_trainer_step_scored(tr.h, _stream(), _text("asg").to_device(), B, T, _ptr(feat), L, _ptr(tgt), _ptr(loss), 3.0,
                                                        _ptr(counts)),
        "null text": lambda: lib.w2l_trainer_step_scored(tr.h, _stream(), None, B, T, _ptr(feat), L, _ptr(tgt), _ptr(loss), 3.0, _ptr(counts)),
        "null counts": lambda: lib.w2l_trainer_step_scored(tr.h, _stream(), dev, B, T, _ptr(feat), L, _ptr(tgt), _ptr(loss), 3.0, None),
        "null target": lambda: lib.w2l_trainer_step_scored(tr.h, _stream(), dev, B, T, _ptr(feat), L, None, _ptr(loss), 3.0, _ptr(counts)),
        "null features": lambda: lib.w2l_trainer_step_scored(tr.h, _stream(), dev, B, T, None, L, _ptr(tgt), _ptr(loss), 3.0, _ptr(counts)),
        "total_batch": lambda: lib.w2l_trainer_step_scored(tr.h, _stream(), dev, B, T, _ptr(feat), L, _ptr(tgt), _ptr(loss), 0.0, _ptr(counts)),
        "target width": lambda: lib.w2l_trainer_step_scored(tr.h, _stream(), dev, B, T, _ptr(feat), wide.shape[1], _ptr(wide), _ptr(loss), 3.0,
                                                            _ptr(counts)),
    }
    for name, call in calls.items():
        launches = lib.w2l_launch_count()
        assert call() == 1, name
        assert "trainer_step_scored" in lib.w2l_last_error().decode(), name
        assert lib.w2l_launch_count() == launches, name
        now = (tr.get_flat(0), tr.get_flat(1), tr.position(), tr.amp_state())
        assert torch.equal(now[0], state[0]) and torch.equal(now[1], state[1]) and now[2:] == state[2:], name
    with pytest.raises(ValueError):
        tr.step(feat, tgt, text=_text("asg"))
    tr.close()
    # a seq2seq trainer is refused by the entry point
    s = s2s.make_trainer(32, 9, maxlen=6, lr=0.05, lrcrit=0.05)
    f2 = s2s.features(rng, 2, 40)
    t2 = torch.zeros((2, 3), dtype=torch.int32, device="cuda")
    before = (s.get_flat(0).clone(), s.position())
    assert lib.w2l_trainer_step_scored(s.h, _stream(), dev, 2, 40, _ptr(f2), 3, _ptr(t2), _ptr(loss), 2.0, _ptr(counts)) == 1
    assert "seq2seq" in lib.w2l_last_error().decode()
    assert torch.equal(s.get_flat(0), before[0]) and s.position() == before[1]
    with pytest.raises(W2LError):
        tr.step(feat, tgt, text=text)  # (closed)
    s.close()
