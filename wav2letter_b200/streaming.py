"""Python handles on the streaming acoustic model (w2l_stream_* in include/w2l_b200.h) and on its MFSC front end
(StreamingFeatures, w2l_mfsc_stream_*), whose features StreamingAM.run takes as they come.

A trained streaming TDS network run chunk by chunk over many concurrent streams, as the in-tree inference library
runs it.  Per stream, the emissions of every `run` and of `finish`, put end to end, do not change by a bit with the
chunking or with the other streams in a call, and match the eval-mode `Trainer.forward` of the whole utterance in
frame count and up to the rounding of the LayerNorm statistics.  The harness owns the tensors; the frame arithmetic
and every kernel run inside libw2l_b200.so.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import capi
from .capi import _check, _ptr, _stream, lib


def _ints(values) -> ctypes.Array:
    v = [int(x) for x in values]
    return (ctypes.c_int * len(v))(*v)


class StreamingAM:
    def __init__(self, trainer, max_streams: int, max_chunk: int = 50, precision: str | None = None):
        """Snapshot of `trainer`'s network parameters (training may go on) with state for `max_streams` slots and chunks
        of at most `max_chunk` feature frames.  precision: None (the thread's w2l_set_precision), "tf32", "f32" or
        "bf16"."""
        saved = capi.get_precision()
        if precision is not None:
            capi.set_precision(precision)
        try:
            h = lib.w2l_stream_create(trainer.h, _stream(), int(max_streams), int(max_chunk))
        finally:
            capi.set_precision(saved)
        if not h:
            raise capi.W2LError(1, lib.w2l_last_error().decode())
        self.h = ctypes.c_void_p(h)
        self.max_streams, self.max_chunk = int(max_streams), int(max_chunk)
        self.n_label = trainer.n_label
        self.max_frames_out = int(lib.w2l_stream_max_frames_out(self.h))

    @property
    def state_bytes(self) -> int:
        """device bytes of carried state per slot"""
        return int(lib.w2l_stream_state_bytes(self.h))

    def start(self, slots):
        """reset the slots; a running slot forgets its past"""
        _check(lib.w2l_stream_start(self.h, _stream(), len(slots), _ints(slots)))

    def run(self, slots, features: torch.Tensor | None, frames=None, finish: bool = False):
        """features: CUDA float [n,1,F,Tc] contiguous (the trainer's layout), frames: valid frames per stream (default
        Tc).  Returns (emissions [n,T'max,N], frames_out list): rows t >= frames_out[i] of stream i are unspecified."""
        n = len(slots)
        if features is None:
            Tc, fptr = 0, None
            frames = [0] * n if frames is None else frames
        else:
            if not features.is_cuda or features.dtype != torch.float32 or not features.is_contiguous() or features.shape[0] != n:
                raise TypeError("features must be a contiguous CUDA float32 tensor [n,1,F,Tc]")
            Tc, fptr = int(features.shape[3]), _ptr(features)
            frames = [Tc] * n if frames is None else frames
        cap = n * self.max_frames_out * self.n_label
        out = torch.empty(max(cap, 1), dtype=torch.float32, device="cuda")
        fo = (ctypes.c_int * n)()
        _check(lib.w2l_stream_run(self.h, _stream(), n, _ints(slots), _ints(frames), fptr, Tc, int(finish), _ptr(out), cap, fo))
        frames_out = list(fo)
        tmax = max(frames_out) if frames_out else 0
        return out[: n * tmax * self.n_label].view(n, tmax, self.n_label), frames_out

    def finish(self, slots, features: torch.Tensor | None = None, frames=None):
        """run the last chunk (may be None: no new frames) and every layer's right padding; the slots stay finished
        until the next start"""
        return self.run(slots, features, frames, finish=True)

    def close(self):
        if getattr(self, "h", None):
            lib.w2l_stream_destroy(self.h)
            self.h = None

    __del__ = close


class StreamingFeatures:
    def __init__(self, max_streams: int, max_chunk_samples: int, n_filters: int = 80, left_ctx: int = 300, sample_rate: int = 16000,
                 frame_ms: int = 25, stride_ms: int = 10):
        """MFSC front end (w2l_mfsc_stream_*) for `max_streams` slots and chunks of at most `max_chunk_samples` samples
        (at most 65535), normalised over the last `left_ctx` frames and the current one (`--localnrmlleftctx`, >= 1).
        Its features are what StreamingAM(trainer, n, max_chunk=self.max_frames_out).run takes."""
        h = lib.w2l_mfsc_stream_create(_stream(), int(max_streams), int(max_chunk_samples), int(sample_rate), int(frame_ms), int(stride_ms),
                                       int(n_filters), int(left_ctx))
        if not h:
            raise capi.W2LError(1, lib.w2l_last_error().decode())
        self.h = ctypes.c_void_p(h)
        self.max_streams, self.max_chunk_samples, self.n_filters = int(max_streams), int(max_chunk_samples), int(n_filters)
        self.sample_rate, self.frame_ms, self.stride_ms, self.left_ctx = int(sample_rate), int(frame_ms), int(stride_ms), int(left_ctx)
        self.max_frames_out = int(lib.w2l_mfsc_stream_max_frames_out(self.h))

    @property
    def state_bytes(self) -> int:
        """device bytes of carried state per slot"""
        return int(lib.w2l_mfsc_stream_state_bytes(self.h))

    def start(self, slots):
        """reset the slots; a running slot forgets its past"""
        _check(lib.w2l_mfsc_stream_start(self.h, _stream(), len(slots), _ints(slots)))

    def run(self, slots, audio: torch.Tensor | None, samples=None, finish: bool = False):
        """audio: CUDA float [n,Sc] contiguous (w2l_mfsc's sample scale), samples: new samples per stream (default Sc).
        Returns (features [n,1,F,Tf], frames list) with Tf = max(frames); frames t >= frames[i] of stream i are 0."""
        n = len(slots)
        if audio is None:
            Sc, aptr = 0, None
            samples = [0] * n if samples is None else samples
        else:
            if not audio.is_cuda or audio.dtype != torch.float32 or not audio.is_contiguous() or audio.dim() != 2 or audio.shape[0] != n:
                raise TypeError("audio must be a contiguous CUDA float32 tensor [n,Sc]")
            Sc, aptr = int(audio.shape[1]), _ptr(audio)
            samples = [Sc] * n if samples is None else samples
        cap = n * self.n_filters * self.max_frames_out
        out = torch.empty(max(cap, 1), dtype=torch.float32, device="cuda")
        fo = (ctypes.c_int * n)()
        _check(lib.w2l_mfsc_stream_run(self.h, _stream(), n, _ints(slots), _ints(samples), aptr, Sc, int(finish), _ptr(out), cap, fo))
        frames = list(fo)
        tf = max(frames) if frames else 0
        return out[: n * self.n_filters * tf].view(n, 1, self.n_filters, tf), frames

    def finish(self, slots, audio: torch.Tensor | None = None, samples=None):
        """run the last chunk (may be None) and drop the remainder; the slots stay finished until the next start"""
        return self.run(slots, audio, samples, finish=True)

    def close(self):
        if getattr(self, "h", None):
            lib.w2l_mfsc_stream_destroy(self.h)
            self.h = None

    __del__ = close


def plan(arch_text: str, n_feat: int, n_label: int, chunks, finish: bool = True, max_convs: int = 64):
    """Host-only frame bookkeeping of one stream (w2l_stream_plan): returns (conv specs [(kw, stride, pad_left,
    pad_right)], output frames [call][conv], held frames [call][conv])."""
    n_calls = len(chunks)
    spec = (ctypes.c_int * (4 * max_convs))()
    out = (ctypes.c_int * max(1, n_calls * max_convs))()
    tails = (ctypes.c_int * max(1, n_calls * max_convs))()
    nc = ctypes.c_int(0)
    _check(lib.w2l_stream_plan(arch_text.encode(), n_feat, n_label, n_calls, _ints(chunks) if n_calls else None, int(finish), max_convs,
                               ctypes.byref(nc), spec, out, tails))
    c = nc.value
    specs = [tuple(spec[4 * k:4 * k + 4]) for k in range(c)]
    o = np.array(out[: n_calls * max_convs], dtype=np.int64).reshape(n_calls, max_convs)[:, :c]
    t = np.array(tails[: n_calls * max_convs], dtype=np.int64).reshape(n_calls, max_convs)[:, :c]
    return specs, o, t
