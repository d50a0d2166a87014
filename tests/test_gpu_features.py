"""w2l_mfsc on the GPU against the float64 NumPy reference (tests/features_reference.py): both frame sizes of the
recipes, 40 and 80 filters, per-utterance and local normalisation, on batches that mix 0.5 s and 33 s utterances with
the edge cases (shorter than a frame, exactly one frame, silence); padding, determinism, causality of the local mode,
and raw audio -> features -> TDS + CTC training end to end."""
import numpy as np
import pytest
import torch

import features_reference as R

pytestmark = pytest.mark.gpu

FS = 16000


def synth(n, seed, amp=2000.0, noise=100.0):
    """speech-like test signal at 16-bit scale: harmonics of a pitch that jumps every 0.1 s, a syllable envelope, noise"""
    rng = np.random.default_rng(seed)
    f0 = np.repeat(rng.uniform(90, 280, n // 1600 + 1), 1600)[:n]
    phase = np.cumsum(2 * np.pi * f0 / FS)
    x = sum(rng.uniform(0.2, 1.0) / h * np.sin(h * phase + rng.uniform(0, 6.3)) for h in range(1, 9))
    env = 0.55 + 0.45 * np.sin(2 * np.pi * np.arange(n) / (FS * 0.37) + rng.uniform(0, 6.3))
    return amp * env * x + rng.normal(0, noise, n)


def batch(frame_ms, seed=0, noise=100.0):
    frame = R.frame_samples(FS, frame_ms)
    lengths = [8000, 33 * FS, frame - 1, frame, 2 * FS, 117353]
    S = max(lengths)
    rng = np.random.default_rng(seed + 100)
    audio = rng.normal(0, 5000.0, (len(lengths), S))  # whatever lies past an utterance's length must be ignored
    for b, n in enumerate(lengths):
        audio[b, :n] = 0.0 if b == 4 else synth(n, seed + b, noise=noise)
    return audio.astype(np.float32), lengths


@pytest.mark.parametrize("left_ctx", [0, 300])
@pytest.mark.parametrize("n_filters", [40, 80])
@pytest.mark.parametrize("frame_ms,stride_ms", [(25, 10), (30, 10)])
def test_mfsc_matches_reference(frame_ms, stride_ms, n_filters, left_ctx):
    from wav2letter_b200.features import mfsc

    audio, lengths = batch(frame_ms)
    feat, frames = mfsc(torch.from_numpy(audio).cuda(), lengths, FS, frame_ms, stride_ms, n_filters, left_ctx)
    torch.cuda.synchronize()
    ref = R.mfsc_batch(audio.astype(np.float64), lengths, FS, frame_ms, stride_ms, n_filters, left_ctx)
    assert frames == [R.num_frames(n, FS, frame_ms, stride_ms) for n in lengths]
    assert frames[2] == 0 and frames[3] == 1
    assert feat.shape == (len(lengths), 1, n_filters, ref.shape[2])
    got = feat[:, 0].cpu().numpy()
    assert np.isfinite(got).all()
    err = np.abs(got - ref).max()
    assert err <= 1e-4, f"max |gpu - ref| = {err}"
    for b, t in enumerate(frames):  # padding frames (and the whole of the empty / silent utterances) are exactly 0
        assert (got[b, :, t:] == 0).all()
    assert (got[2] == 0).all() and (got[4] == 0).all()


def test_mfsc_near_the_mel_floor():
    """The DFT runs in fp32-accurate arithmetic, so its error is fp32-grade relative to each frame's strongest bins.
    With a noise floor of 30 under voicing of amplitude 2000, the lowest filters of some frames sit about 80 dB below
    the frame's peak, near the mel floor, and single elements differ from float64 by up to about 1.4e-4 (NumPy's
    float32 path: 2.1e-4 on the same batch)."""
    from wav2letter_b200.features import mfsc

    audio, lengths = batch(30, noise=30.0)
    feat, _ = mfsc(torch.from_numpy(audio).cuda(), lengths, FS, 30, 10, 80, 0)
    ref = R.mfsc_batch(audio.astype(np.float64), lengths, FS, 30, 10, 80, 0)
    err = np.abs(feat[:, 0].cpu().numpy() - ref)
    assert err.max() <= 3e-4 and np.quantile(err, 0.9999) <= 3e-5, (err.max(), np.quantile(err, 0.9999))


def test_mfsc_is_deterministic_and_ignores_the_precision_setting():
    from wav2letter_b200 import capi
    from wav2letter_b200.features import mfsc

    audio, lengths = batch(25, seed=7)
    a = torch.from_numpy(audio).cuda()
    one, _ = mfsc(a, lengths, left_ctx=300)
    two, _ = mfsc(a, lengths, left_ctx=300)
    assert torch.equal(one, two)
    prev = capi.get_precision()
    try:
        for p in ("tf32", "bf16"):
            capi.set_precision(p)
            assert torch.equal(mfsc(a, lengths, left_ctx=300)[0], one)
    finally:
        capi.set_precision(prev)


def test_local_normalisation_is_causal():
    from wav2letter_b200.features import mfsc

    x = synth(20 * FS, 11).astype(np.float32)
    whole, (tw,) = mfsc(torch.from_numpy(x[None]).cuda(), [len(x)], n_filters=80, left_ctx=300)
    n = 124321
    part, (tp,) = mfsc(torch.from_numpy(x[None, :n].copy()).cuda(), [n], n_filters=80, left_ctx=300)
    assert tp == R.num_frames(n, FS, 25, 10) and tp < tw
    assert float((part[..., :tp] - whole[..., :tp]).abs().max()) <= 1e-6


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


def test_audio_to_trained_model():
    """tone-sequence "utterances" (token k = a 0.2 s tone at 300 * 1.2^k Hz) -> mfsc(F = 40) -> TDS + CTC"""
    from wav2letter_b200.features import mfsc
    from wav2letter_b200.trainer import Trainer

    rng = np.random.default_rng(5)
    B, L, N = 4, 5, 12  # 11 tokens + the CTC blank
    seg = FS // 5
    tgt = rng.integers(0, N - 1, (B, L)).astype(np.int32)
    t = np.arange(seg) / FS
    ramp = np.minimum(1.0, np.minimum(t, t[::-1]) / 0.01)
    audio = np.stack([np.concatenate([3000 * ramp * np.sin(2 * np.pi * 300 * 1.2 ** k * t) for k in row]) for row in tgt])
    audio = (audio + rng.normal(0, 20.0, audio.shape)).astype(np.float32)
    feat, frames = mfsc(torch.from_numpy(audio).cuda(), [audio.shape[1]] * B, n_filters=40)
    assert feat.shape == (B, 1, 40, frames[0]) and frames[0] == 98
    tr = Trainer(ARCH_F40, 40, N, "ctc", "none", lr=0.02, momentum=0.5, maxgradnorm=5.0)
    y = torch.from_numpy(tgt).cuda()
    first = tr.step(feat, y, train=False).sum().item()
    for _ in range(40):
        tr.step(feat, y, train=True)
    last = tr.step(feat, y, train=False).sum().item()
    tr.close()
    assert np.isfinite(last) and last < 0.7 * first, (first, last)
