"""MFSC (log-mel filterbank) features on the GPU: raw audio -> the trainer's [B,1,F,T] input (w2l_mfsc in
include/w2l_b200.h; DESIGN.md §4 "Features")."""
from __future__ import annotations

import ctypes

import torch

from .capi import _check, _ptr, _req, _stream, lib, workspace


def num_frames(n_samples: int, sample_rate: int = 16000, frame_ms: int = 25, stride_ms: int = 10) -> int:
    """Frames of an utterance of n_samples samples: 0 below one frame, else 1 + (n - frame) // stride."""
    n = int(lib.w2l_mfsc_num_frames(int(n_samples), int(sample_rate), int(frame_ms), int(stride_ms)))
    if n < 0:
        raise ValueError(lib.w2l_last_error().decode())
    return n


def mfsc(audio: torch.Tensor, lengths, sample_rate: int = 16000, frame_ms: int = 25, stride_ms: int = 10,
         n_filters: int = 80, left_ctx: int = 0):
    """audio: CUDA float32 [B, max_samples] (16-bit sample scale), lengths: samples per utterance (host ints).
    Returns (features CUDA float32 [B,1,F,T] with T the longest utterance's frame count and zero padding behind each
    utterance, frames per utterance as a list).  left_ctx = 0 normalises per utterance, > 0 over the last left_ctx
    frames and the current one (`--localnrmlleftctx`)."""
    audio = _req(audio, torch.float32, "audio")
    if audio.dim() != 2:
        raise ValueError("audio: expected [B, max_samples]")
    B, S = audio.shape
    n = [int(v) for v in (lengths.tolist() if torch.is_tensor(lengths) else lengths)]
    if len(n) != B:
        raise ValueError(f"lengths: expected {B} entries, got {len(n)}")
    frames = [num_frames(v, sample_rate, frame_ms, stride_ms) for v in n]
    T = max(frames, default=0)
    feat = torch.empty((B, 1, int(n_filters), T), dtype=torch.float32, device=audio.device)
    host_n = (ctypes.c_int32 * B)(*n)
    ws = workspace(lib.w2l_mfsc_workspace_size(B, S, sample_rate, frame_ms, stride_ms, n_filters), audio.device)
    _check(lib.w2l_mfsc(_stream(), B, S, _ptr(audio), host_n, int(sample_rate), int(frame_ms), int(stride_ms), int(n_filters),
                        int(left_ctx), _ptr(feat) if T > 0 else None, T, _ptr(ws), ws.numel()))
    return feat, frames
