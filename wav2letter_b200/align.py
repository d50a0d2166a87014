"""Forced alignment to word timings: raw audio + transcripts -> `.align` lines (one per utterance,
`id<TAB>seg\\nseg...`, each segment "id 1 <begin s> <duration s> <word>", silence as "$"; DESIGN.md §3
"Forced alignment").  Audio decoding is the caller's: the audio arrives as float samples at 16-bit scale."""
from __future__ import annotations

import torch

from .features import mfsc


def align_lines(trainer, text, audio: torch.Tensor, n_samples, transcripts, ids, sample_rate: int = 16000,
                frame_ms: int = 25, stride_ms: int = 10, n_filters: int = 80, left_ctx: int = 0):
    """trainer: a Trainer (CTC, ASG or LinSeg); text: the TextPipeline its targets were made with; audio CUDA float32
    [B, max_samples]; n_samples, transcripts, ids: one entry per utterance.  Returns one line per utterance (no
    newline), or None for an utterance whose transcript cannot be aligned in its frames."""
    feat, _ = mfsc(audio, n_samples, sample_rate, frame_ms, stride_ms, n_filters, left_ctx)
    target = text.encode_batch(transcripts)
    _, idx = trainer.align(feat, torch.from_numpy(target).to(audio.device))
    idx = idx.cpu().numpy()
    ms_per_frame = stride_ms * trainer.time_stride()
    return [None if idx[b, 0] < 0 else text.align_words(target[b], idx[b], ms_per_frame, ids[b])
            for b in range(len(transcripts))]
