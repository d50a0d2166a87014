"""Python handle on the C++ training-step driver (w2l_trainer_* in include/w2l_b200.h).

The harness owns device memory (torch tensors) and the launch (torchrun); every arithmetic step of the
training loop runs inside libw2l_b200.so.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import capi
from .capi import _check, _ptr, _stream, lib


class Trainer:
    def __init__(self, arch_text: str, n_feat: int, n_label: int, criterion: str = "ctc", scale_mode="none",
                 transdiag: float = 0.0, lr: float = 0.05, lrcrit: float = 0.0, momentum: float = 0.0,
                 maxgradnorm: float = 0.0, precision: str | None = None, seq2seq: dict | None = None):
        """precision: None (the thread's w2l_set_precision), "tf32", "f32" (fp32-accurate), "bf16" or "fp16".
        criterion "seq2seq" takes its settings from `seq2seq` (Train.cpp's flags): hidden (--encoderdim), eos, pad,
        maxdecoderoutputlen, and optionally rounds (--decoderattnround, 1), layers (--decoderrnnlayer, 1), dropout
        (--decoderdropout, 0), labelsmooth (0), pctteacherforcing (100), window_std (--softwstd; 0 = no window) and
        train_with_window (--trainWithWindow, False); n_label counts the dictionary with eos and pad."""
        mode = capi.SCALE_MODES[scale_mode] if isinstance(scale_mode, str) else int(scale_mode)
        if criterion == "seq2seq":
            s = dict(SEQ2SEQ_DEFAULTS, **(seq2seq or {}))
            self.h = lib.w2l_trainer_create_seq2seq(_stream(), arch_text.encode(), n_feat, n_label, int(s["hidden"]), int(s["eos"]), int(s["pad"]),
                                                    int(s["maxdecoderoutputlen"]), int(s["rounds"]), int(s["layers"]), float(s["dropout"]),
                                                    float(s["labelsmooth"]), int(s["pctteacherforcing"]), float(s["window_std"]),
                                                    int(bool(s["train_with_window"])), lr, lrcrit, momentum, maxgradnorm)
        else:
            self.h = lib.w2l_trainer_create(_stream(), arch_text.encode(), n_feat, n_label, criterion.encode(), mode,
                                            transdiag, lr, lrcrit, momentum, maxgradnorm)
        if not self.h:
            raise capi.W2LError(1, lib.w2l_last_error().decode())
        self.h = ctypes.c_void_p(self.h)
        self.n_feat, self.n_label, self.criterion = n_feat, n_label, criterion
        if precision is not None:
            self.set_precision(precision)

    def set_precision(self, precision):
        _check(lib.w2l_trainer_set_precision(self.h, capi.PRECISIONS[precision] if isinstance(precision, str) else int(precision)))

    INT64_MAX = (1 << 63) - 1

    def set_schedule(self, warmup: int = 1, gamma: float = 1.0, stepsize: int = INT64_MAX, lrcosine: bool = False,
                     nbatches: int = INT64_MAX, lr_decay: int = INT64_MAX, lr_decay_step: int = INT64_MAX):
        """Train.cpp's learning-rate schedule (--warmup --gamma --stepsize --lrcosine --iter --lr_decay --lr_decay_step),
        applied to the base rates at every training step; the defaults leave the rates unchanged"""
        _check(lib.w2l_trainer_set_schedule(self.h, int(warmup), float(gamma), int(stepsize), int(bool(lrcosine)), int(nbatches),
                                            int(lr_decay), int(lr_decay_step)))

    def set_position(self, update: int, epoch: int):
        """updates already taken (Train.cpp's curBatch before the next step) and the running epoch (curEpoch, 1-based)"""
        _check(lib.w2l_trainer_set_position(self.h, int(update), int(epoch)))

    def position(self) -> tuple[int, int]:
        u, e = ctypes.c_longlong(0), ctypes.c_longlong(0)
        _check(lib.w2l_trainer_position(self.h, ctypes.byref(u), ctypes.byref(e)))
        return int(u.value), int(e.value)

    def set_lr(self, lr: float, lrcrit: float):
        """the base learning rates of the network and the criterion (the schedule scales them)"""
        _check(lib.w2l_trainer_set_lr(self.h, float(lr), float(lrcrit)))

    def lr(self) -> tuple[float, float]:
        """the learning rates the next training step uses"""
        a, b = ctypes.c_float(0), ctypes.c_float(0)
        _check(lib.w2l_trainer_lr(self.h, ctypes.byref(a), ctypes.byref(b)))
        return float(a.value), float(b.value)

    def set_amp(self, on: bool = True, initial_scale: float = 4096.0, update_interval: int = 2000, max_scale: float = 32000.0,
                min_scale: float = 1e-4):
        """Train.cpp's dynamic loss scaling (--fl_amp_use_mixed_precision and its --fl_amp_* flags; the defaults are theirs)"""
        _check(lib.w2l_trainer_set_amp(self.h, int(bool(on)), float(initial_scale), int(update_interval), float(max_scale), float(min_scale)))

    def amp_state(self) -> tuple[float, int, int]:
        """(loss scale of the next step, attempt counter, retried attempts so far)"""
        s, c, r = ctypes.c_double(0), ctypes.c_int(0), ctypes.c_longlong(0)
        _check(lib.w2l_trainer_amp_state(self.h, _stream(), ctypes.byref(s), ctypes.byref(c), ctypes.byref(r)))
        return float(s.value), int(c.value), int(r.value)

    def set_grad_stream(self, on: bool):
        """True (default): the Linear layers' weight gradients run on a second stream beside the data-gradient chain"""
        _check(lib.w2l_trainer_set_grad_stream(self.h, int(on)))

    def set_grad_stream_delay(self, us: int):
        """tests: hold the gradient stream back by `us` microseconds before each piece of work handed to it"""
        _check(lib.w2l_trainer_set_grad_stream_delay(self.h, int(us)))

    def skipped_steps(self) -> int:
        """steps whose update the device-side guard skipped (NaN / Inf loss or gradient); synchronises"""
        n = ctypes.c_longlong(0)
        _check(lib.w2l_trainer_status(self.h, _stream(), ctypes.byref(n)))
        return int(n.value)

    def save(self, path: str):
        """own-format checkpoint: constructor arguments + parameter / momentum arenas, position, learning-rate schedule and loss
        scaling
        (Train.cpp:747-800)"""
        _check(lib.w2l_trainer_save(self.h, _stream(), path.encode()))

    @classmethod
    def load(cls, path: str) -> "Trainer":
        h = lib.w2l_trainer_load(_stream(), path.encode())
        if not h:
            raise capi.W2LError(1, lib.w2l_last_error().decode())
        self = cls.__new__(cls)
        self.h = ctypes.c_void_p(h)
        self.n_feat = self.n_label = self.criterion = None
        return self

    def export_streaming(self, outdir: str, tokens_text: str | None = None):
        """arrays of every layer in the layouts of the in-tree streaming inference library + transitions.bin / tokens.txt
        (the conversions of recipes/streaming_convnets/tools/StreamingTDSModelConverter.cpp)"""
        _check(lib.w2l_trainer_export_streaming(self.h, _stream(), outdir.encode(), None if tokens_text is None else tokens_text.encode()))

    def close(self):
        if getattr(self, "h", None):
            lib.w2l_trainer_destroy(self.h)
            self.h = None

    __del__ = close

    def describe(self) -> str:
        return lib.w2l_trainer_describe(self.h).decode()

    def num_params(self, which: int = 0) -> int:
        """which: 0 the network, 1 the criterion, 2 the teacher (set_ema; without one, the network)"""
        return int(lib.w2l_trainer_num_params(self.h, which))

    def layout(self, which: int = 0):
        """[(offset, elements, dims)] of every parameter inside the flat arena (16-byte aligned slots)."""
        n = 4096
        el = (ctypes.c_longlong * n)()
        dims = (ctypes.c_longlong * (4 * n))()
        cnt = lib.w2l_trainer_param_layout(self.h, which, n, el, dims)
        if cnt < 0:
            raise capi.W2LError(capi.W2L_ERR_INVALID_ARGUMENT, lib.w2l_last_error().decode())
        out, off = [], 0
        for i in range(cnt):
            out.append((off, int(el[i]), tuple(int(dims[4 * i + d]) for d in range(4))))
            off += (int(el[i]) + 3) // 4 * 4
        return out

    def get_flat(self, which: int = 0, what: int = 0) -> torch.Tensor:
        n = self.num_params(which)
        out = torch.empty(max(n, 1), dtype=torch.float32, device="cuda")
        _check(lib.w2l_trainer_get_flat(self.h, _stream(), which, what, _ptr(out)))
        return out[:n]

    def set_flat(self, flat: torch.Tensor, which: int = 0):
        _check(lib.w2l_trainer_set_flat(self.h, _stream(), which, _ptr(flat.contiguous())))

    def step(self, features: torch.Tensor, target: torch.Tensor, train: bool = True, total_batch: float | None = None,
             loss_out: torch.Tensor | None = None, input_sizes=None, target_sizes=None, text=None):
        """features: CUDA float [B,1,F,T] contiguous (== ArrayFire [T,F,1,B]); target CUDA int32 [B,L].
        total_batch: the batch summed over ranks (default B); every gradient is divided by it.  A training step raises
        W2LError (code 1) before running anything unless it is finite and > 0; an eval step does not use it.
        input_sizes / target_sizes (seq2seq only; a list or a CUDA int32 tensor of B entries): the input frame counts of a
        padded batch (the counts features.mfsc returns) and the target sizes (tokens plus eos).  Utterance b then attends
        to its first ceil(d_b T' / max d) encoder frames, and the soft window follows its own diagonal.

        text: a TextPipeline (ctc for a ctc trainer, asg for asg and linseg) makes this a scored training step, Train.cpp's
        meters.train (:1699-1714): returns (loss, counts), counts CUDA int32 [B, 8] laid out as TextPipeline.edit_counts,
        scoring the criterion's viterbi path of THIS step's training-mode output (dropout and SpecAugment included)
        against target.  Loss, gradients and update are those of the unscored step, bit for bit; the path and scoring run
        beside the backward and add no host read.  Add counts to an ErrorRates; under mixed precision Train.cpp adds them
        once per attempt, i.e. 1 + the step's increase of amp_state()[2] times (a retried attempt replays its random draws,
        so every attempt's counts are the same).  Which batches to score (--pcttraineval, a hash of the sample ids) is the
        caller's loop, like data loading; counts stay per rank.  Not for seq2seq (its path is the greedy decode)."""
        B, _, F, T = features.shape
        if text is not None:
            return self._step_scored(features, target, train, total_batch, loss_out, input_sizes, target_sizes, text)
        L = target.shape[1]
        isz, tsz = size_arg(input_sizes, B, "input_sizes"), size_arg(target_sizes, B, "target_sizes")
        if loss_out is None:
            loss_out = torch.empty(B, dtype=torch.float32, device=features.device)
        tb = float(total_batch if total_batch is not None else B)
        if isz is None and tsz is None:
            _check(lib.w2l_trainer_step(self.h, _stream(), B, T, _ptr(features), L, _ptr(target), _ptr(loss_out), int(train), tb))
        else:
            _check(lib.w2l_trainer_step_sized(self.h, _stream(), B, T, _ptr(features), L, _ptr(target), _ptr(isz), _ptr(tsz), _ptr(loss_out),
                                              int(train), tb))
        return loss_out

    def _step_scored(self, features, target, train, total_batch, loss_out, input_sizes, target_sizes, text):
        """step(text=...): its arguments are checked here, before anything runs"""
        from .text import TextPipeline

        if not isinstance(text, TextPipeline):
            raise TypeError("text: expected a TextPipeline")
        if not train:
            raise ValueError("text: a scored step is a training step (train=True); score eval batches with evaluate")
        if input_sizes is not None or target_sizes is not None:
            raise ValueError("text: input_sizes / target_sizes are the seq2seq criterion's, which a scored step does not cover")
        if self.criterion == "seq2seq":
            raise ValueError("text: the seq2seq criterion's viterbi path is its greedy decode, which a training step does not run")
        want = {"ctc": "ctc", "asg": "asg", "linseg": "asg"}.get(self.criterion)  # (None for a loaded trainer: the C side checks)
        if want is not None and text.criterion != want:
            raise ValueError(f"text: a {self.criterion} trainer is scored with a {want} TextPipeline, got {text.criterion}")
        B = features.shape[0]
        if target.dim() != 2 or target.shape[0] != B:
            raise ValueError(f"target: expected [B={B}, L], got {tuple(target.shape)}")
        target = capi._req(target, torch.int32, "target")
        loss_out = capi._req(loss_out, torch.float32, "loss_out")
        if loss_out is None:
            loss_out = torch.empty(B, dtype=torch.float32, device=features.device)
        elif loss_out.numel() != B:
            raise ValueError(f"loss_out: expected {B} elements, got {loss_out.numel()}")
        counts = torch.empty((B, 8), dtype=torch.int32, device=features.device)
        tb = float(total_batch if total_batch is not None else B)
        _check(lib.w2l_trainer_step_scored(self.h, _stream(), text.to_device(), B, features.shape[3], _ptr(features), target.shape[1],
                                           _ptr(target), _ptr(loss_out), tb, _ptr(counts)))
        return loss_out, counts

    def output_width(self) -> int:
        """features per frame of the network output: n_label, or 2 * hidden (the encoder) for seq2seq"""
        w = ctypes.c_int(0)
        _check(lib.w2l_trainer_output_width(self.h, ctypes.byref(w)))
        return int(w.value)

    def forward(self, features: torch.Tensor, teacher: bool = False) -> torch.Tensor:
        """eval-mode network output [B, T', width]; teacher=True: the teacher's (set_ema; without one, the network's),
        slimIPL's soft pseudo-labels"""
        B, _, F, T = features.shape
        width = self.output_width()

        def call(out, cap, tout):
            if teacher:
                return lib.w2l_trainer_forward_teacher(self.h, _stream(), B, T, _ptr(features), 1, _ptr(out), cap, tout)
            return lib.w2l_trainer_forward(self.h, _stream(), B, T, _ptr(features), _ptr(out), cap, tout)

        (out,), t = _frame_results(call, features, width, torch.float32)
        return out.view(B, t, width)

    def set_ema(self, decay: float | None = 0.999):
        """slimIPL's teacher (--slimIPL_ema --slimIPL_ema_decay): a second copy of the network, started from the network as
        it is now, that every later training step moves by ema = ema * decay + net * (1 - decay).  None drops it."""
        _check(lib.w2l_trainer_set_ema(self.h, _stream(), 0 if decay is None else 1, 0.0 if decay is None else float(decay)))

    def ema(self) -> float | None:
        """the teacher's decay, or None without a teacher"""
        on, d = ctypes.c_int(0), ctypes.c_double(0)
        _check(lib.w2l_trainer_ema(self.h, ctypes.byref(on), ctypes.byref(d)))
        return float(d.value) if on.value else None

    def viterbi_path(self, features: torch.Tensor, teacher: bool = False, input_sizes=None) -> torch.Tensor:
        """crit->viterbiPath of the eval-mode output of the network or (teacher=True) the teacher: CUDA int32 [B, T'] (CTC
        per-frame argmax, ASG / LinSeg FCC Viterbi) or [B, maxdecoderoutputlen] (seq2seq greedy decode, padded with pad).
        input_sizes: seq2seq only, as in step."""
        B, _, F, T = features.shape
        isz = size_arg(input_sizes, B, "input_sizes")
        try:
            maxlen = self.seq2seq_config()["maxdecoderoutputlen"]
        except capi.W2LError:  # not seq2seq: one token per output frame
            maxlen = 0

        def call(path, cap, tout):
            return lib.w2l_trainer_viterbi_path(self.h, _stream(), B, T, _ptr(features), _ptr(isz), int(bool(teacher)), _ptr(path), cap, tout)

        (path,), t = _frame_results(call, features, frames=maxlen)
        return path.view(B, t)

    def evaluate(self, features: torch.Tensor, target: torch.Tensor, text, input_sizes=None, target_sizes=None):
        """Train.cpp's test() on one batch: the eval-mode forward, the criterion's loss (the bits of step(train=False)), its
        viterbi path (as viterbi_path) and the device scoring of that path against target (TextPipeline.edit_counts).
        text: the batch's TextPipeline.  input_sizes / target_sizes: seq2seq only, as in step.  Returns CUDA tensors
        (loss float32 [B], counts int32 [B, 8]); nothing is read back to the host but the greedy decode's own polls."""
        from .text import TextPipeline

        if not isinstance(text, TextPipeline):
            raise TypeError("text: expected a TextPipeline")
        B, _, F, T = features.shape
        target = capi._req(target, torch.int32, "target")
        L = target.shape[1]
        isz, tsz = size_arg(input_sizes, B, "input_sizes"), size_arg(target_sizes, B, "target_sizes")
        loss = torch.empty(B, dtype=torch.float32, device=features.device)
        counts = torch.empty((B, 8), dtype=torch.int32, device=features.device)
        _check(lib.w2l_trainer_evaluate(self.h, _stream(), text.to_device(), B, T, _ptr(features), L, _ptr(target), _ptr(isz), _ptr(tsz),
                                        _ptr(loss), _ptr(counts)))
        return loss, counts

    def step_soft(self, features: torch.Tensor, teacher_logits: torch.Tensor, soft_scale: float = 1.0, total_batch: float | None = None,
                  loss_out: torch.Tensor | None = None) -> torch.Tensor:
        """slimIPL's training step on an unlabelled batch with soft pseudo-labels (--slimIPL_use_soft): the loss is
        soft_scale * -mean over frames of sum_c softmax(teacher_logits)_c logSoftmax(output)_c, teacher_logits CUDA float32
        [B, T', width] as forward returns it.  total_batch defaults to the world size (the loss is one scalar per rank).
        Returns the loss, CUDA float32 [1]."""
        B, _, F, T = features.shape
        teacher_logits = capi._req(teacher_logits, torch.float32, "teacher_logits")
        if teacher_logits.dim() != 3 or teacher_logits.shape[0] != B or teacher_logits.shape[2] != self.output_width():
            raise ValueError(f"teacher_logits: expected [B={B}, T', {self.output_width()}], got {tuple(teacher_logits.shape)}")
        if loss_out is None:
            loss_out = torch.empty(1, dtype=torch.float32, device=features.device)
        if total_batch is None:
            total_batch = torch.distributed.get_world_size() if torch.distributed.is_available() and torch.distributed.is_initialized() else 1
        _check(lib.w2l_trainer_step_soft(self.h, _stream(), B, T, _ptr(features), _ptr(teacher_logits), teacher_logits.shape[1],
                                         float(soft_scale), _ptr(loss_out), float(total_batch)))
        return loss_out

    def seq2seq_config(self) -> dict:
        """hidden, eos, pad, maxdecoderoutputlen, rounds, layers and whether the window is still set (seq2seq only)"""
        v = (ctypes.c_int * 7)()
        _check(lib.w2l_trainer_seq2seq_config(self.h, v))
        return dict(zip(("hidden", "eos", "pad", "maxdecoderoutputlen", "rounds", "layers", "window_set"), (int(x) for x in v)))

    def clear_window(self):
        """Seq2SeqCriterion::clearWindow(): after the --pretrainWindow updates, train without the soft window"""
        _check(lib.w2l_trainer_clear_window(self.h))

    def seq2seq_seed(self) -> int:
        """the Philox seed the last training step's criterion drew (token substitution; dropout after layer k: seed + 1 + k)"""
        s = ctypes.c_ulonglong(0)
        _check(lib.w2l_trainer_seq2seq_seed(self.h, ctypes.byref(s)))
        return int(s.value)

    def decode(self, features: torch.Tensor, input_sizes=None):
        """Greedy decode (seq2seq): eval-mode forward, then argmax token by token from startEmbedding until eos or
        maxdecoderoutputlen steps.  Returns (tokens CUDA int32 [B, maxdecoderoutputlen] padded with pad, lengths CUDA int32 [B]).
        input_sizes: as in step, so that each utterance of a padded batch decodes over its own frames."""
        B, _, F, T = features.shape
        isz = size_arg(input_sizes, B, "input_sizes")
        n = self.seq2seq_config()["maxdecoderoutputlen"]
        tokens = torch.empty((B, n), dtype=torch.int32, device=features.device)
        lengths = torch.empty(B, dtype=torch.int32, device=features.device)
        if isz is None:
            _check(lib.w2l_trainer_decode(self.h, _stream(), B, T, _ptr(features), _ptr(tokens), _ptr(lengths), tokens.numel()))
        else:
            _check(lib.w2l_trainer_decode_sized(self.h, _stream(), B, T, _ptr(features), _ptr(isz), _ptr(tokens), _ptr(lengths), tokens.numel()))
        return tokens, lengths

    def beam_search(self, features: torch.Tensor, beam_size: int = 4, max_len: int | None = None, input_sizes=None):
        """Beam search (seq2seq): eval-mode forward, then Seq2SeqCriterion::beamSearchBatch over the batch with beam_size
        in [1, 16] for at most max_len steps (None: maxdecoderoutputlen).  Returns CUDA tensors (tokens int32 [B, K, L]
        padded with pad, lengths int32 [B, K], scores float32 [B, K], counts int32 [B]): per utterance the completed
        hypotheses if any (best first once more than K completed, else in completion order), otherwise the live beam at
        length L.  Slots at or beyond counts[b] hold pad, length 0 and score -inf.  input_sizes: as in decode."""
        B, _, F, T = features.shape
        isz = size_arg(input_sizes, B, "input_sizes")
        L = int(max_len) if max_len is not None else self.seq2seq_config()["maxdecoderoutputlen"]
        K = int(beam_size)
        dev = features.device
        tokens = torch.empty((B, max(K, 1), max(L, 1)), dtype=torch.int32, device=dev)
        lengths = torch.empty((B, max(K, 1)), dtype=torch.int32, device=dev)
        scores = torch.empty((B, max(K, 1)), dtype=torch.float32, device=dev)
        counts = torch.empty(B, dtype=torch.int32, device=dev)
        if isz is None:
            _check(lib.w2l_trainer_beam_search(self.h, _stream(), B, T, _ptr(features), K, L, _ptr(tokens), _ptr(lengths), _ptr(scores),
                                               _ptr(counts), tokens.numel()))
        else:
            _check(lib.w2l_trainer_beam_search_sized(self.h, _stream(), B, T, _ptr(features), _ptr(isz), K, L, _ptr(tokens), _ptr(lengths),
                                                     _ptr(scores), _ptr(counts), tokens.numel()))
        return tokens, lengths, scores, counts

    def align(self, features: torch.Tensor, target: torch.Tensor):
        """Forced alignment: eval-mode forward, then the criterion's viterbiPathWithTarget.  features CUDA float
        [B,1,F,T], target CUDA int32 [B,L] (-1 padded).  Returns (path, idx), CUDA int32 [B,T']: the token per output
        frame and, for CTC, the extended-target state, for ASG, the target position (-1 over a row that cannot be
        aligned)."""
        B, _, F, T = features.shape
        L = target.shape[1]

        def call(path, idx, cap, tout):
            return lib.w2l_trainer_align(self.h, _stream(), B, T, _ptr(features), L, _ptr(target), _ptr(path), _ptr(idx), cap, tout)

        (path, idx), t = _frame_results(call, features, buffers=2)
        return path.view(B, t), idx.view(B, t)

    def time_stride(self) -> int:
        """input frames per output frame (the product of the network's time strides)"""
        return int(lib.w2l_trainer_time_stride(self.h))

    def sync_parameters(self):
        _check(lib.w2l_trainer_sync_parameters(self.h, _stream()))


def _frame_results(call, features: torch.Tensor, width: int = 1, dtype=torch.int32, buffers: int = 1, frames: int = 0):
    """The [B][T'][width] results of the eval entry points that report T' through t_out (forward, viterbi_path, align):
    call(*buffers, capacity, t_out) fills `buffers` tensors of capacity elements each and returns the status.  They are
    first sized for max(2T + 64, frames) frames (SAME-padded even kernels grow the frame count by one each) and, when
    explicit padding (e.g. 170 frames a side) makes T' larger, once more at the T' the first call reported.
    Returns (the buffers cut to B T' width elements, T')."""
    B, T = features.shape[0], features.shape[3]
    tout = ctypes.c_int(0)

    def run(n):
        bufs = [torch.empty(B * n * width, dtype=dtype, device=features.device) for _ in range(buffers)]
        return call(*bufs, B * n * width, ctypes.byref(tout)), bufs

    n = max(2 * T + 64, frames)
    rc, bufs = run(n)
    if rc != 0 and tout.value > n:
        rc, bufs = run(tout.value)
    _check(rc)
    return [b[: B * tout.value * width] for b in bufs], tout.value


def size_arg(sizes, B: int, name: str):
    """None, or the per-utterance sizes as a contiguous CUDA int32 tensor of B entries: from a list / tuple of whole
    numbers, or a CUDA int32 tensor as it is.  Their values are checked on the device (a bad one gives that utterance a
    NaN loss); their form is checked here, before anything runs."""
    if sizes is None:
        return None
    if isinstance(sizes, torch.Tensor):
        if not sizes.is_cuda or sizes.dtype != torch.int32 or not sizes.is_contiguous() or sizes.dim() != 1:
            raise TypeError(f"{name}: expected a contiguous 1-d CUDA tensor of torch.int32")
        t = sizes
    else:
        vals = list(sizes)
        if not all(isinstance(v, (int, np.integer)) and not isinstance(v, bool) for v in vals):
            raise TypeError(f"{name}: expected whole numbers")
        if any(v < -(1 << 31) or v >= (1 << 31) for v in vals):
            raise ValueError(f"{name}: values must fit in int32")
        t = None
    n = t.numel() if t is not None else len(vals)
    if n != B:
        raise ValueError(f"{name}: {n} entries for a batch of {B}")
    return t if t is not None else torch.tensor(vals, dtype=torch.int32, device="cuda")


def nccl_unique_id() -> bytes:
    buf = ctypes.create_string_buffer(128)
    _check(lib.w2l_nccl_unique_id(buf))
    return buf.raw


def init_distributed(rank: int, world: int, uid: bytes):
    _check(lib.w2l_init_distributed(rank, world, ctypes.c_char_p(uid)))


# the seq2seq settings' defaults (Train.cpp's flag defaults where they exist)
SEQ2SEQ_DEFAULTS = dict(rounds=1, layers=1, dropout=0.0, labelsmooth=0.0, pctteacherforcing=100, window_std=0.0, train_with_window=False)

from . import archs  # noqa: E402

# recipes/seq2seq_tds/librispeech/network.arch with the CTC head BASELINE.json configs[1] asks for
# (last line `L 1440 NLABEL` instead of the seq2seq encoder's `L 1440 1024`)
SEQ2SEQ_TDS_CTC_ARCH = archs.seq2seq_tds(ctc_head=True)


def conv_glu_librispeech_arch() -> str:
    """recipes/conv_glu/librispeech/network.arch (17 WeightNorm Conv1D+GLU layers, two WeightNorm Linear layers)"""
    return archs.conv_glu_librispeech()
