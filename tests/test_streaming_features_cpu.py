"""CPU checks of the streaming MFSC front end (w2l_mfsc_stream_* in include/w2l_b200.h): the symbols, create's argument
checks (they run before any CUDA call), and the oracle the GPU tests use — a NumPy transcription of LogMelFeature::run's
sample buffer chained with the StreamingLocalNorm transcription equals the whole-utterance reference in any chunking."""
import ctypes
import os

import numpy as np
import pytest

import features_reference as R
from test_features_cpu import StreamingLocalNorm

FS = 16000
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("w2l_mfsc_stream_create", "w2l_mfsc_stream_destroy", "w2l_mfsc_stream_state_bytes", "w2l_mfsc_stream_max_frames_out",
           "w2l_mfsc_stream_start", "w2l_mfsc_stream_run")


class LogMelBuffer:
    """LogMelFeature::run (inference/module/feature/LogMelFeature.cpp:42-65): append the samples, frame what is held
    (avail < frame ? 0 : 1 + (avail - frame) / stride frames), consume frames * stride samples and keep the rest;
    finish drops the remainder (no right padding).  Returns the log-mel frames [n, F] in float64."""

    def __init__(self, p: R.Params):
        self.p, self.buf = p, np.zeros(0)

    def run(self, x, finish=False):
        self.buf = np.concatenate([self.buf, np.asarray(x, dtype=np.float64)])
        avail, frame, stride = len(self.buf), self.p.frame, self.p.stride
        fr = R.frames_of(self.buf, frame, stride)
        assert len(fr) == (0 if avail < frame else 1 + (avail - frame) // stride)
        out = np.log(np.maximum(R.magnitude(self.p, fr) @ self.p.fbank_t, R.MEL_FLOOR))
        self.buf = np.zeros(0) if finish else self.buf[len(fr) * self.p.stride:]
        assert len(self.buf) < self.p.frame
        return out


def stream_reference(p, x, cuts, left_ctx):
    """x fed in the pieces between `cuts`, the last one finishing: (features [T, F] float32, frames per call)"""
    mel, norm = LogMelBuffer(p), StreamingLocalNorm(p.n_filters, left_ctx)
    parts, frames = [], []
    pieces = list(zip(cuts[:-1], cuts[1:]))
    for k, (a, b) in enumerate(pieces):
        f = mel.run(x[a:b], finish=k == len(pieces) - 1)
        frames.append(len(f))
        parts.append(norm.run(f.astype(np.float32)))
    return np.concatenate(parts), frames


def speech(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / FS
    f0 = np.repeat(rng.uniform(90, 280, n // 1600 + 1), 1600)[:n]
    x = sum(np.sin(np.cumsum(2 * np.pi * h * f0 / FS)) / h for h in range(1, 6))
    return 2000 * (0.55 + 0.45 * np.sin(2 * np.pi * t / 0.37)) * x + rng.normal(0, 100, n)


def test_symbols_in_header_prototypes_and_library():
    from wav2letter_b200 import capi

    header = open(os.path.join(ROOT, "include", "w2l_b200.h")).read()
    for s in SYMBOLS:
        assert s + "(" in header and s in capi.PROTOTYPES and hasattr(capi.lib, s)


def test_create_rejects_bad_arguments_before_any_cuda_call():
    from wav2letter_b200 import capi

    lib = capi.lib

    def create(S=4, C=8000, fs=FS, fms=25, sms=10, F=80, left=300):
        return lib.w2l_mfsc_stream_create(None, S, C, fs, fms, sms, F, left)

    for kw, text in ((dict(left=0), b"left_ctx"), (dict(left=-1), b"left_ctx"),
                     (dict(fs=22050), b"multiple of 4"), (dict(F=257), b"256 filters"), (dict(fms=200), b"2048 samples"),
                     (dict(S=0), b"max_streams"), (dict(S=1025), b"max_streams"),
                     (dict(C=0), b"max_chunk_samples"), (dict(C=65536), b"max_chunk_samples"),
                     (dict(F=0), b"positive"), (dict(sms=0), b"positive")):
        assert create(**kw) is None, kw
        assert text in lib.w2l_last_error(), (kw, lib.w2l_last_error())
    assert lib.w2l_mfsc_stream_state_bytes(None) == -1 and lib.w2l_mfsc_stream_max_frames_out(None) == -1
    one = (ctypes.c_int * 1)(0)
    assert lib.w2l_mfsc_stream_start(None, None, 1, one) == 1 and b"null handle" in lib.w2l_last_error()


@pytest.mark.parametrize("left_ctx", [1, 7, 300])
def test_buffer_transcription_chained_with_localnorm_equals_the_utterance_reference(left_ctx):
    p = R.Params(FS, 25, 10, 40)
    n = 24000 + 123
    x = speech(n, left_ctx)
    whole = R.mfsc_utterance(p, x, left_ctx)
    rng = np.random.default_rng(left_ctx)
    fixed = [0, 0, 1, p.frame - 1, p.frame, 8000, 160, 0]  # empty calls, one sample, below / exactly a frame, 0.5 s
    for trial in range(3):
        sizes = fixed if trial == 0 else [int(v) for v in rng.integers(0, 3000, 40)]
        cuts = np.minimum(np.concatenate([[0], np.cumsum(sizes)]), n)
        cuts = list(cuts[cuts < n]) + [n]
        got, frames = stream_reference(p, x, cuts, left_ctx)
        assert sum(frames) == whole.shape[0] == R.num_frames(n, FS, 25, 10)
        np.testing.assert_allclose(got, whole, atol=2e-4)
    # the remainder a finish drops: fewer than a frame's samples after the last frame
    assert (n - p.frame) % p.stride > 0
