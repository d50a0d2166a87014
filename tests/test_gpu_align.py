"""Forced alignment on the GPU: w2l_ctc_viterbi_target bit for bit against the NumPy contract
(tests/ctc_align_reference.py) over every states-per-lane width (S up to 2047), T up to 4000, N = 30 and 10 000,
batches of 1, 16 and 64 with repeated labels, integer-valued emissions (ties), empty and infeasible targets; the
collapse of every path; determinism; and, end to end, TDS + CTC / ASG models trained on a synthetic tone task:
Trainer.align against the reference on Trainer.forward's emissions, ASG's viterbiPathWithTarget against
w2l_fac_viterbi, and align_lines (audio -> `.align` lines) holding every transcript word once, in order."""
import numpy as np
import pytest
import torch

import ctc_align_reference as R

pytestmark = pytest.mark.gpu


def make_targets(rng, B, T, N, L):
    """[B, L] targets: full length with repeats, random shorter ones, an empty one, an infeasible one, one that needs
    exactly T frames when it fits"""
    y = rng.integers(0, N - 1, (B, L)).astype(np.int32)
    rep = rng.random((B, L)) < 0.15
    for b in range(B):
        for l in range(1, L):
            if rep[b, l]:
                y[b, l] = y[b, l - 1]
        n = L if b % 4 == 0 else int(rng.integers(0, L + 1))
        y[b, n:] = -1
    if B > 1:
        y[1, :] = -1  # empty
    if B > 2 and L >= 2:  # repeats push it past T when L is close to T, else exactly feasible
        y[2, :] = 0
        y[2, min(L, T) :] = -1
    return y


def emissions(rng, B, T, N, integer):
    if integer:  # few distinct values: ties everywhere
        return torch.from_numpy(rng.integers(-2, 3, (B, T, N)).astype(np.float32))
    return torch.from_numpy(rng.normal(0, 2, (B, T, N)).astype(np.float32))


def check(e, y):
    from wav2letter_b200 import capi

    path, state = capi.ctc_viterbi_target(e.cuda(), torch.from_numpy(y).cuda(), return_state=True)
    rp, rs = R.ctc_viterbi_target(e.numpy(), y)
    assert torch.equal(path.cpu(), torch.from_numpy(rp)), "path differs from the reference"
    assert torch.equal(state.cpu(), torch.from_numpy(rs)), "state differs from the reference"
    N = e.shape[2]
    T = e.shape[1]
    for b in range(y.shape[0]):
        tgt = y[b, : R.target_size(y[b])]
        feasible = len(tgt) + int(np.sum(tgt[1:] == tgt[:-1])) <= T and np.all((tgt >= 0) & (tgt < N - 1))
        if feasible:
            assert R.collapse(rp[b], N - 1) == tgt.tolist()
        else:
            assert (rp[b] == -1).all()
    return path, state


# (B, T, N, L, integer emissions): every states-per-lane width P = 1 .. 64 (Sp = 32 P >= 2 min(L, T) + 1)
CASES = [
    (64, 60, 30, 15, True),      # P = 1
    (64, 100, 30, 31, False),    # P = 2
    (16, 200, 30, 63, True),     # P = 4
    (16, 300, 30, 127, False),   # P = 8
    (64, 500, 30, 255, True),    # P = 16
    (16, 1500, 30, 511, True),   # P = 32
    (1, 4000, 30, 1023, False),  # P = 64, S = 2047
    (16, 200, 10000, 66, False),
    (1, 4000, 10000, 1023, True),
    (16, 40, 30, 64, False),     # L > T: P from min(L, T); most targets infeasible
]


@pytest.mark.parametrize("B,T,N,L,integer", CASES)
def test_matches_reference(B, T, N, L, integer):
    rng = np.random.default_rng(B * 7919 + T * 31 + N + L)
    e = emissions(rng, B, T, N, integer)
    y = make_targets(rng, B, T, N, L)
    if B >= 16 and L <= T:
        y[3, :] = rng.integers(0, N - 1, L)
        y[3, 1::2] = y[3, 0::2][: L // 2]  # every label repeated: needs 1.5 L frames
    check(e, y)


def test_exactly_feasible_and_one_frame():
    rng = np.random.default_rng(3)
    e = emissions(rng, 3, 7, 5, True)
    y = np.array([[0, 0, 1, 1, -1], [0, 1, 2, 3, 0], [2, 2, 2, 2, -1]], np.int32)  # 6, 5 and 7 frames needed
    check(e, y)
    check(emissions(rng, 4, 1, 5, False), np.array([[0], [-1], [3], [4]], np.int32))  # T = 1; blank as label


def test_deterministic():
    from wav2letter_b200 import capi

    rng = np.random.default_rng(11)
    e = emissions(rng, 16, 800, 30, True).cuda()
    y = torch.from_numpy(make_targets(rng, 16, 800, 30, 300)).cuda()
    a = capi.ctc_viterbi_target(e, y, return_state=True)
    b = capi.ctc_viterbi_target(e, y, return_state=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_time_stride_follows_the_arch():
    from wav2letter_b200 import archs
    from wav2letter_b200.trainer import Trainer

    for arch, F, stride in ((archs.seq2seq_tds(True), 80, 8), (archs.streaming_tds(), 80, 8), (archs.conv_glu_librispeech(), 40, 1),
                            (ARCH_F40, 40, 4)):
        tr = Trainer(arch, F, 30, "ctc")
        assert tr.time_stride() == stride
        tr.close()


ARCH_F40 = """V -1 NFEAT 1 0
C2 1 4 5 1 2 1 -1 -1
R
DO 0.0
LN 3
TDS 4 5 40 0.0
C2 4 8 5 1 2 1 -1 -1
R
DO 0.0
LN 3
TDS 8 5 40 0.0
TDS 8 5 40 0.0
V 0 320 1 0
RO 1 0 3 2
L 320 NLABEL
"""
FS = 16000
LETTERS = "abcdefg"
TOKENS = "|\n" + "\n".join(LETTERS) + "\n"  # | a..g


def tone_task(rng, B, text):
    """transcripts of 3 words of 1-3 letters; every letter is 0.2 s of a tone at 300 * 1.25^k Hz (letter k), every word
    is followed by 0.2 s of near-silence"""
    transcripts = [" ".join("".join(rng.choice(list(LETTERS), rng.integers(1, 4))) for _ in range(3)) for _ in range(B)]
    seg = FS // 5
    t = np.arange(seg) / FS
    ramp = np.minimum(1.0, np.minimum(t, t[::-1]) / 0.01)
    tone = {c: 3000 * ramp * np.sin(2 * np.pi * 300 * 1.25 ** k * t) for k, c in enumerate(LETTERS)}
    pieces = [np.concatenate([np.concatenate([tone[c] for c in w] + [np.zeros(seg)]) for w in tr.split()]) for tr in transcripts]
    S = max(len(p) for p in pieces)
    audio = np.zeros((B, S))
    for b, p in enumerate(pieces):
        audio[b, : len(p)] = p
    audio = (audio + rng.normal(0, 20.0, audio.shape)).astype(np.float32)
    return transcripts, text.encode_batch(transcripts), audio, [S] * B


@pytest.mark.parametrize("criterion", ["ctc", "asg"])
def test_trained_model_alignment_end_to_end(criterion):
    from wav2letter_b200 import capi
    from wav2letter_b200.align import align_lines
    from wav2letter_b200.features import mfsc
    from wav2letter_b200.text import TextPipeline
    from wav2letter_b200.trainer import Trainer

    rng = np.random.default_rng(21)
    # ASG targets drop adjacent repeats unless they are packed into replabels
    text = TextPipeline(TOKENS, "", criterion, 1 if criterion == "asg" else 0, "", False, "|")
    N = text.num_classes
    B = 8
    transcripts, target, audio, n_samples = tone_task(rng, B, text)
    dev_audio = torch.from_numpy(audio).cuda()
    feat, _ = mfsc(dev_audio, n_samples, n_filters=40)
    y = torch.from_numpy(target).cuda()
    tr = Trainer(ARCH_F40, 40, N, criterion, "none", transdiag=2.0 if criterion == "asg" else 0.0, lr=0.02, lrcrit=0.002,
                 momentum=0.5, maxgradnorm=5.0)
    first = tr.step(feat, y, train=False).sum().item()
    for _ in range(60):
        tr.step(feat, y, train=True)
    last = tr.step(feat, y, train=False).sum().item()
    assert np.isfinite(last) and last < 0.7 * first, (first, last)

    emis = tr.forward(feat).contiguous()
    path, idx = tr.align(feat, y)
    assert path.shape == emis.shape[:2] and idx.shape == emis.shape[:2]
    if criterion == "ctc":
        rp, rs = R.ctc_viterbi_target(emis.cpu().numpy(), target)
        assert torch.equal(path.cpu(), torch.from_numpy(rp)) and torch.equal(idx.cpu(), torch.from_numpy(rs))
    else:
        trans = tr.get_flat(which=1)[: N * N].view(N, N).contiguous()
        fp, fi = capi.fac_viterbi(emis, y, trans, return_index=True)
        assert torch.equal(path, fp) and torch.equal(idx, fi)
    assert (idx >= 0).all()

    assert tr.time_stride() == 4
    lines = align_lines(tr, text, dev_audio, n_samples, transcripts, [f"utt{b}" for b in range(B)], n_filters=40)
    dur = n_samples[0] / FS
    for b, line in enumerate(lines):
        utt, rest = line.split("\t")
        assert utt == f"utt{b}"
        segs = [s.split() for s in rest.strip().split("\\n")]
        assert all(len(s) == 5 and s[0] == utt for s in segs) and segs[0][4] == "$"
        words = [s[4] for s in segs if s[4] != "$"]
        assert words == transcripts[b].split()
        ends = 0.0
        for s in segs:
            begin, length = float(s[2]), float(s[3])
            assert begin >= ends - 1e-6 and length >= 0
            ends = begin + length
        assert ends <= emis.shape[1] * 0.04 + 1e-6 and ends >= dur - 0.2
    tr.close()
