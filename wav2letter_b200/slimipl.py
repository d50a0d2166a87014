"""slimIPL's pseudo-labels (recipes/slimIPL/src/Train.cpp:1362-1415): what the trainer's loop turns an unlabelled batch
into before its step.  The cache policies (--slimIPL_type) and the interleaving of labelled and unlabelled batches are
the caller's loop, like data loading (DESIGN.md §7)."""
from __future__ import annotations

import numpy as np
import torch


def pl_strings(text, paths) -> list:
    """Train.cpp's hard PL text of every row of host token paths: tokenToWord(path, true) (prediction -> letters ->
    words), joined by spaces"""
    return [" ".join(text.ltr2wrd(text.prediction2ltr(row))) for row in np.asarray(paths, dtype=np.int32)]


def pseudo_labels(trainer, text, features: torch.Tensor, input_sizes=None):
    """hard PLs of a batch: the teacher's viterbiPath, copied to the host (afToVector, :1380), through pl_strings and
    back into targets with the dataset's transform (text.encode_batch).  Returns (targets CUDA int32 [B, L] padded with
    text.pad_index, target sizes CUDA int32 [B] (tokens, eos included for seq2seq), the PL strings)."""
    strings = pl_strings(text, trainer.viterbi_path(features, teacher=True, input_sizes=input_sizes).cpu().numpy())
    targets = text.encode_batch(strings)
    sizes = (targets != text.pad_index).sum(axis=1).astype(np.int32)
    return torch.from_numpy(targets).to(features.device), torch.from_numpy(sizes).to(features.device), strings


def soft_targets(trainer, features: torch.Tensor) -> torch.Tensor:
    """soft PLs of a batch (--slimIPL_use_soft, :1413-1415): the teacher's raw eval-mode output [B, T', width], the
    teacher_logits of Trainer.step_soft"""
    return trainer.forward(features, teacher=True)
