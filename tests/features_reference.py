"""NumPy restatement of the MFSC features w2l_mfsc computes (DESIGN.md §4 "Features"), float64 by default.

The settings the reference pins in its own tree: LogMelFeature::init (recipes/streaming_convnets/inference/inference/
module/feature/LogMelFeature.cpp:75-91) and Train.cpp:288-290 — no zero-mean frame, no dither, no energy coefficient,
magnitude (not power) spectrum, filters between 0 Hz and fs/2.  The constants marked RECALLED are flashlight
FeatureParams / Mfsc defaults; flashlight is not vendored, so they are written from memory, not read from source.
"""
from __future__ import annotations

import numpy as np

PREEMPH = 0.97      # RECALLED: FeatureParams::preemCoef
MEL_FLOOR = 1.0     # RECALLED: FeatureParams::melFloor, applied as log(max(x, MEL_FLOOR))
STD_FLOOR = 1e-5    # LocalNorm.cpp kEpsilon (and, RECALLED, the per-utterance normalize threshold)


def frame_samples(sample_rate: int, ms: int) -> int:
    """round(sample_rate * ms / 1000), halves up (RECALLED: FeatureParams::numFrameSizeSamples)"""
    return (int(sample_rate) * int(ms) + 500) // 1000


def num_frames(n: int, sample_rate: int, frame_ms: int, stride_ms: int) -> int:
    frame, stride = frame_samples(sample_rate, frame_ms), frame_samples(sample_rate, stride_ms)
    return 0 if n < frame else 1 + (n - frame) // stride


def nfft_for(frame: int) -> int:
    n = 1
    while n < frame:
        n <<= 1
    return n


def mel(hz):
    """HTK mel scale"""
    return 2595.0 * np.log10(1.0 + np.asarray(hz, dtype=np.float64) / 700.0)


def mel_inv(m):
    return 700.0 * (10.0 ** (np.asarray(m, dtype=np.float64) / 2595.0) - 1.0)


def filter_edges(n_filters: int, bins: int, sample_rate: int) -> np.ndarray:
    """the n_filters + 2 triangle corners in bin units: mel^-1(i * dmel) * (bins - 1) * 2 / fs"""
    dmel = mel(sample_rate / 2.0) / (n_filters + 1)
    return mel_inv(np.arange(n_filters + 2) * dmel) * (bins - 1) * 2.0 / sample_rate


def filterbank(n_filters: int, bins: int, sample_rate: int) -> np.ndarray:
    """[F][bins]: weight of bin i in filter f = max(0, min(rising, falling))"""
    e = filter_edges(n_filters, bins, sample_rate)
    i = np.arange(bins, dtype=np.float64)[None, :]
    lo, c, hi = e[:-2, None], e[1:-1, None], e[2:, None]
    return np.maximum(0.0, np.minimum((i - lo) / (c - lo), (hi - i) / (hi - c)))


def hamming(n: int) -> np.ndarray:
    return 0.54 - 0.46 * np.cos(2.0 * np.pi * np.arange(n) / (n - 1))


def preemphasis(frames: np.ndarray) -> np.ndarray:
    """x[i] -= 0.97 x[i-1] for i descending to 1, then x[0] *= 0.03, per frame (rows)"""
    y = frames.copy()
    y[:, 1:] -= PREEMPH * frames[:, :-1]
    y[:, 0] *= 1.0 - PREEMPH
    return y


def folded_basis(frame: int, nfft: int) -> np.ndarray:
    """[2 * bins][frame]: row 2k / 2k+1 maps a raw frame to Re / -Im of bin k of rfft(hamming * preemphasis(frame), nfft)
    — the B' operand of the GPU's DFT GEMM"""
    bins = nfft // 2 + 1
    i = np.arange(frame)
    ang = 2.0 * np.pi * ((np.arange(bins)[:, None] * i[None, :]) % nfft) / nfft
    w = hamming(frame)
    basis = np.empty((2 * bins, frame))
    for r, trig in ((0, np.cos), (1, np.sin)):
        t = w[None, :] * trig(ang)                # window * e_k(i)
        b = t.copy()
        b[:, 0] *= 1.0 - PREEMPH
        b[:, :-1] -= PREEMPH * t[:, 1:]          # sample m also enters y[m+1] with weight -0.97
        basis[r::2] = b
    return basis


def frames_of(x: np.ndarray, frame: int, stride: int) -> np.ndarray:
    n = len(x)
    if n < frame:
        return np.zeros((0, frame), dtype=x.dtype)
    t = 1 + (n - frame) // stride
    return np.lib.stride_tricks.sliding_window_view(x, frame)[: (t - 1) * stride + 1: stride]


class Params:
    def __init__(self, sample_rate=16000, frame_ms=25, stride_ms=10, n_filters=80, dtype=np.float64):
        self.sample_rate, self.n_filters = sample_rate, n_filters
        self.frame, self.stride = frame_samples(sample_rate, frame_ms), frame_samples(sample_rate, stride_ms)
        self.nfft = nfft_for(self.frame)
        self.bins = self.nfft // 2 + 1
        self.dtype = dtype
        self.basis_t = np.ascontiguousarray(folded_basis(self.frame, self.nfft).T.astype(dtype))   # [frame][2 bins]
        self.fbank_t = np.ascontiguousarray(filterbank(n_filters, self.bins, sample_rate).T.astype(dtype))  # [bins][F]


def magnitude(p: Params, frames: np.ndarray) -> np.ndarray:
    """|spectrum| [T][bins] through the folded basis"""
    c = frames.astype(p.dtype, copy=False) @ p.basis_t
    return np.sqrt(c[:, 0::2] ** 2 + c[:, 1::2] ** 2)


def log_mel(p: Params, x: np.ndarray) -> np.ndarray:
    """[T][F] log(max(mel, 1)) of one utterance"""
    fr = frames_of(np.asarray(x, dtype=p.dtype), p.frame, p.stride)
    return np.log(np.maximum(magnitude(p, fr) @ p.fbank_t, p.dtype(MEL_FLOOR)))


def normalize_utterance(f: np.ndarray) -> np.ndarray:
    """mean / population std over all T x F values (RECALLED: the per-utterance normalize of the reference's loader)"""
    if f.size == 0:
        return f
    m = f.mean(dtype=np.float64)
    sd = np.sqrt(max(float((f.astype(np.float64) ** 2).mean()) - m * m, 0.0))
    return ((f - m) / (sd if sd > STD_FLOOR else 1.0)).astype(f.dtype)


def normalize_local(f: np.ndarray, left_ctx: int) -> np.ndarray:
    """frame t over frames max(0, t - left_ctx) .. t (LocalNorm::run with no right context)"""
    T, F = f.shape
    if T == 0:
        return f
    s1 = np.concatenate([[0.0], np.cumsum(f.sum(1, dtype=np.float64))])
    s2 = np.concatenate([[0.0], np.cumsum((f.astype(np.float64) ** 2).sum(1))])
    t = np.arange(T)
    lo = np.maximum(0, t - left_ctx)
    cnt = (t - lo + 1) * F
    m = (s1[t + 1] - s1[lo]) / cnt
    sd = np.sqrt(np.maximum((s2[t + 1] - s2[lo]) / cnt - m * m, 0.0))
    sd = np.where(sd <= STD_FLOOR, 1.0, sd)
    return ((f - m[:, None]) / sd[:, None]).astype(f.dtype)


def mfsc_utterance(p: Params, x: np.ndarray, left_ctx: int = 0) -> np.ndarray:
    """[T][F] normalised features of one utterance"""
    f = log_mel(p, x)
    return normalize_local(f, left_ctx) if left_ctx > 0 else normalize_utterance(f)


def mfsc_batch(audio, lengths, sample_rate=16000, frame_ms=25, stride_ms=10, n_filters=80, left_ctx=0,
               dtype=np.float64) -> np.ndarray:
    """[B][F][T_max] (= the trainer's [B,1,F,T] without the singleton), zero behind each utterance"""
    p = Params(sample_rate, frame_ms, stride_ms, n_filters, dtype)
    feats = [mfsc_utterance(p, np.asarray(a)[:n], left_ctx) for a, n in zip(audio, lengths)]
    T = max((f.shape[0] for f in feats), default=0)
    out = np.zeros((len(feats), n_filters, T), dtype=dtype)
    for b, f in enumerate(feats):
        out[b, :, : f.shape[0]] = f.T
    return out
