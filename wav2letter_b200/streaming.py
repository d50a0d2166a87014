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


class _StreamHandle:
    """What both runtimes' handles share: the w2l_<api>_* life cycle, start, finish and the slot and count side of run."""
    _api = ""  # "stream" or "mfsc_stream"

    def _open(self, h):
        if not h:
            raise capi.W2LError(1, lib.w2l_last_error().decode())
        self.h = ctypes.c_void_p(h)
        self.max_frames_out = int(self._fn("max_frames_out")(self.h))

    def _fn(self, name: str):
        return getattr(lib, f"w2l_{self._api}_{name}")

    @property
    def state_bytes(self) -> int:
        """device bytes of carried state per slot"""
        return int(self._fn("state_bytes")(self.h))

    def start(self, slots):
        """reset the slots; a running slot forgets its past"""
        _check(self._fn("start")(self.h, _stream(), len(slots), _ints(slots)))

    def _run(self, slots, ptr, chunk: int, counts, finish: bool, per_frame: int):
        """w2l_<api>_run on `counts` new frames or samples per stream (default: all `chunk` of them), into an output of
        max_frames_out frames of `per_frame` floats per stream.  Returns (the output up to the longest stream's frames,
        flat; that frame count; the frames of every stream)."""
        n = len(slots)
        counts = [chunk] * n if counts is None else counts
        cap = n * self.max_frames_out * per_frame
        out = torch.empty(max(cap, 1), dtype=torch.float32, device="cuda")
        fo = (ctypes.c_int * n)()
        _check(self._fn("run")(self.h, _stream(), n, _ints(slots), _ints(counts), ptr, chunk, int(finish), _ptr(out), cap, fo))
        frames = list(fo)
        tmax = max(frames) if frames else 0
        return out[: n * tmax * per_frame], tmax, frames

    def finish(self, slots, *args, **kwargs):
        """run(slots, ...) on the last chunk (default None: no new data), then the end of the stream; the slots stay
        finished until the next start"""
        return self.run(slots, *args, **kwargs, finish=True)

    def close(self):
        if getattr(self, "h", None):
            self._fn("destroy")(self.h)
            self.h = None

    __del__ = close


class StreamingAM(_StreamHandle):
    """The streaming acoustic model; its finish runs every layer's right padding."""
    _api = "stream"

    def __init__(self, trainer, max_streams: int, max_chunk: int = 50, precision: str | None = None):
        """Snapshot of `trainer`'s network parameters (training may go on) with state for `max_streams` slots and chunks
        of at most `max_chunk` feature frames.  precision: None (the thread's w2l_set_precision), "tf32", "f32",
        "bf16" or "fp16"."""
        saved = capi.get_precision()
        if precision is not None:
            capi.set_precision(precision)
        try:
            h = lib.w2l_stream_create(trainer.h, _stream(), int(max_streams), int(max_chunk))
        finally:
            capi.set_precision(saved)
        self.max_streams, self.max_chunk = int(max_streams), int(max_chunk)
        self.n_label = trainer.n_label
        self._open(h)

    def run(self, slots, features: torch.Tensor | None = None, frames=None, finish: bool = False):
        """features: CUDA float [n,1,F,Tc] contiguous (the trainer's layout), frames: valid frames per stream (default
        Tc).  Returns (emissions [n,T'max,N], frames_out list): rows t >= frames_out[i] of stream i are unspecified."""
        n = len(slots)
        if features is None:
            Tc, fptr = 0, None
        else:
            if not features.is_cuda or features.dtype != torch.float32 or not features.is_contiguous() or features.shape[0] != n:
                raise TypeError("features must be a contiguous CUDA float32 tensor [n,1,F,Tc]")
            Tc, fptr = int(features.shape[3]), _ptr(features)
        out, tmax, frames_out = self._run(slots, fptr, Tc, frames, finish, self.n_label)
        return out.view(n, tmax, self.n_label), frames_out


class StreamingFeatures(_StreamHandle):
    """The MFSC front end; its finish drops the remainder, fewer samples than a frame."""
    _api = "mfsc_stream"

    def __init__(self, max_streams: int, max_chunk_samples: int, n_filters: int = 80, left_ctx: int = 300, sample_rate: int = 16000,
                 frame_ms: int = 25, stride_ms: int = 10):
        """MFSC front end (w2l_mfsc_stream_*) for `max_streams` slots and chunks of at most `max_chunk_samples` samples
        (at most 65535), normalised over the last `left_ctx` frames and the current one (`--localnrmlleftctx`, >= 1).
        Its features are what StreamingAM(trainer, n, max_chunk=self.max_frames_out).run takes."""
        h = lib.w2l_mfsc_stream_create(_stream(), int(max_streams), int(max_chunk_samples), int(sample_rate), int(frame_ms), int(stride_ms),
                                       int(n_filters), int(left_ctx))
        self.max_streams, self.max_chunk_samples, self.n_filters = int(max_streams), int(max_chunk_samples), int(n_filters)
        self.sample_rate, self.frame_ms, self.stride_ms, self.left_ctx = int(sample_rate), int(frame_ms), int(stride_ms), int(left_ctx)
        self._open(h)

    def run(self, slots, audio: torch.Tensor | None = None, samples=None, finish: bool = False):
        """audio: CUDA float [n,Sc] contiguous (w2l_mfsc's sample scale), samples: new samples per stream (default Sc).
        Returns (features [n,1,F,Tf], frames list) with Tf = max(frames); frames t >= frames[i] of stream i are 0."""
        n = len(slots)
        if audio is None:
            Sc, aptr = 0, None
        else:
            if not audio.is_cuda or audio.dtype != torch.float32 or not audio.is_contiguous() or audio.dim() != 2 or audio.shape[0] != n:
                raise TypeError("audio must be a contiguous CUDA float32 tensor [n,Sc]")
            Sc, aptr = int(audio.shape[1]), _ptr(audio)
        out, tf, frames = self._run(slots, aptr, Sc, samples, finish, self.n_filters)
        return out.view(n, 1, self.n_filters, tf), frames


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
