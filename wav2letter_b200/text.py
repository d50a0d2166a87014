"""Python handle on the token / target pipeline (w2l_text_* in include/w2l_b200.h; C++ in host/text_pipeline.cpp):
the dataset's target transform and evalOutput's path -> letters -> words -> edit distance (Train.cpp:236-254,296-316,829-872)."""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import capi
from .capi import lib


class TextPipeline:
    def __init__(self, tokens_text: str, lexicon_text: str = "", criterion: str = "ctc", replabel: int = 0, surround: str = "",
                 usewordpiece: bool = False, wordsep: str = "|"):
        h = lib.w2l_text_create(tokens_text.encode(), lexicon_text.encode(), criterion.encode(), int(replabel), surround.encode(),
                                int(usewordpiece), wordsep.encode())
        if not h:
            raise capi.W2LError(1, lib.w2l_last_error().decode())
        self.h = ctypes.c_void_p(h)
        self.criterion = criterion

    def close(self):
        if getattr(self, "dev", None):
            lib.w2l_text_device_destroy(self.dev)
            self.dev = None
        if getattr(self, "h", None):
            lib.w2l_text_destroy(self.h)
            self.h = None

    def to_device(self):
        """builds (once) the device tables w2l_text_edit_counts and Trainer.evaluate read; returns their handle"""
        if getattr(self, "dev", None) is None:
            d = lib.w2l_text_device_create(self.h, capi._stream())
            if not d:
                raise capi.W2LError(1, lib.w2l_last_error().decode())
            self.dev = ctypes.c_void_p(d)
        return self.dev

    def edit_counts(self, paths, targets, path_lengths=None):
        """evalOutput's scoring of a batch on the GPU: paths CUDA int32 [B, n] (viterbi_path / decode rows, a beam_search
        row, slimIPL teacher paths), targets CUDA int32 [B, L] (padded as encode_batch pads), path_lengths None or CUDA
        int32 [B] (row b is then its first path_lengths[b] entries).  Returns CUDA int32 [B, 8]: {reference letters,
        deletions, insertions, substitutions} for letters, then the same for words, equal to prediction2ltr / target2ltr
        / ltr2wrd / EditDistanceMeter on every row; -1 in all eight where those raise (a token outside the dictionary)."""
        paths = capi._req(paths, torch.int32, "paths")
        targets = capi._req(targets, torch.int32, "targets")
        path_lengths = capi._req(path_lengths, torch.int32, "path_lengths")
        if paths.dim() != 2 or targets.dim() != 2 or paths.shape[0] != targets.shape[0]:
            raise ValueError(f"paths [B, n] and targets [B, L] expected, got {tuple(paths.shape)} and {tuple(targets.shape)}")
        B, n = paths.shape
        L = targets.shape[1]
        if path_lengths is not None and tuple(path_lengths.shape) != (B,):
            raise ValueError(f"path_lengths: expected [{B}], got {tuple(path_lengths.shape)}")
        dev = self.to_device()
        counts = torch.empty((B, 8), dtype=torch.int32, device=paths.device)
        nbytes = lib.w2l_text_edit_workspace_size(dev, B, n, L)
        ws = torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=paths.device)
        capi._check(lib.w2l_text_edit_counts(dev, capi._stream(), B, n, capi._ptr(paths), capi._ptr(path_lengths), L, capi._ptr(targets),
                                             capi._ptr(counts), capi._ptr(ws), int(nbytes)))
        return counts

    __del__ = close

    @property
    def num_classes(self) -> int:
        return int(lib.w2l_text_num_classes(self.h))

    def _need(self, n):
        if n < 0:
            raise capi.W2LError(1, lib.w2l_last_error().decode())
        return int(n)

    def encode(self, transcript: str) -> np.ndarray:
        n = self._need(lib.w2l_text_encode(self.h, transcript.encode(), None, 0))
        out = np.zeros(max(n, 1), np.int32)
        lib.w2l_text_encode(self.h, transcript.encode(), out.ctypes.data_as(ctypes.c_void_p), n)
        return out[:n]

    @property
    def pad_index(self) -> int:
        """the value targets are padded with: the pad token's index for seq2seq (the dictionary's last entry), else -1"""
        return self.num_classes - 1 if self.criterion == "seq2seq" else -1

    def encode_batch(self, transcripts) -> np.ndarray:
        """[B][L] int32 padded with pad_index (-1, kTargetPadValue; the pad token for seq2seq)"""
        rows = [self.encode(t) for t in transcripts]
        L = max(1, max(len(r) for r in rows))
        out = np.full((len(rows), L), self.pad_index, np.int32)
        for b, r in enumerate(rows):
            out[b, :len(r)] = r
        return out

    def _str(self, fn, arr) -> list:
        arr = np.ascontiguousarray(arr, dtype=np.int32)
        p = arr.ctypes.data_as(ctypes.c_void_p)
        n = self._need(fn(self.h, p, arr.size, None, 0))
        buf = ctypes.create_string_buffer(n)
        fn(self.h, p, arr.size, buf, n)
        return buf.value.decode().split()

    def prediction2ltr(self, path) -> list:
        return self._str(lib.w2l_text_prediction2ltr, path)

    def target2ltr(self, target_row) -> list:
        return self._str(lib.w2l_text_target2ltr, target_row)

    def ltr2wrd(self, letters) -> list:
        s = " ".join(letters).encode()
        n = self._need(lib.w2l_text_ltr2wrd(self.h, s, None, 0))
        buf = ctypes.create_string_buffer(n)
        lib.w2l_text_ltr2wrd(self.h, s, buf, n)
        return buf.value.decode().split()

    def align_words(self, target_row, idx, ms_per_frame: float, utt_id: str) -> str:
        """one `.align` line (no newline) from a forced alignment: target_row the padded target, idx the aligned index of
        every frame (Trainer.align; CTC: extended-target state, ASG: target position)"""
        tgt = np.ascontiguousarray(target_row, dtype=np.int32)
        ix = np.ascontiguousarray(idx, dtype=np.int32)
        args = (self.h, tgt.ctypes.data_as(ctypes.c_void_p), tgt.size, ix.ctypes.data_as(ctypes.c_void_p), ix.size,
                float(ms_per_frame), utt_id.encode())
        n = self._need(lib.w2l_text_align_words(*args, None, 0))
        buf = ctypes.create_string_buffer(n)
        lib.w2l_text_align_words(*args, buf, n)
        return buf.value.decode()


class EditDistanceMeter:
    """fl::EditDistanceMeter: add(hypothesis tokens, reference tokens); value() = [error %, n, ins %, del %, sub %]"""

    def __init__(self):
        self.acc = (ctypes.c_longlong * 4)(0, 0, 0, 0)  # n, ndel, nins, nsub

    def add(self, hyp, ref):
        capi._check(lib.w2l_edit_distance(" ".join(hyp).encode(), " ".join(ref).encode(), self.acc))

    def value(self):
        n, ndel, nins, nsub = (int(v) for v in self.acc)
        d = float(max(n, 1))
        return [100.0 * (ndel + nins + nsub) / d, n, 100.0 * nins / d, 100.0 * ndel / d, 100.0 * nsub / d]

    def raw(self):
        return tuple(int(v) for v in self.acc)


class ErrorRates:
    """Sums the counts of edit_counts / Trainer.evaluate batch by batch on the device (mtr.tknEdit and mtr.wrdEdit) and
    reports them as EditDistanceMeter.value() does.  Rows of -1 (utterances the host pipeline would refuse) are counted
    in `rejected` and left out of the sums.  Summing across ranks is the caller's: all-reduce `sums` before reading."""

    def __init__(self, device="cuda"):
        self.sums = torch.zeros(9, dtype=torch.int64, device=device)  # 8 counts, then rejected rows

    def add(self, counts: torch.Tensor):
        ok = counts[:, 0] >= 0
        self.sums[:8] += (counts.to(torch.int64) * ok.unsqueeze(1)).sum(0)
        self.sums[8] += (~ok).sum()

    def _value(self, n, ndel, nins, nsub):
        d = float(max(n, 1))
        return [100.0 * (ndel + nins + nsub) / d, n, 100.0 * nins / d, 100.0 * ndel / d, 100.0 * nsub / d]

    def value(self):
        """(token meter value, word meter value, rejected rows); each value is [error %, n, ins %, del %, sub %]"""
        s = [int(v) for v in self.sums.tolist()]
        return self._value(*s[0:4]), self._value(*s[4:8]), s[8]

    def ter(self) -> float:
        return self.value()[0][0]

    def wer(self) -> float:
        return self.value()[1][0]
