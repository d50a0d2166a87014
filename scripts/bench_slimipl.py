"""slimIPL's steps on the TDS + CTC workload of DESIGN.md §6, in one process.

Workload: bench.py's tds_ctc (archs.seq2seq_tds(ctc_head=True), CTC over N = 10 000 classes, B = 16 utterances of 1200
frames, 80 filterbanks, fp32-accurate precision, labelled targets of 30-60 tokens), with a teacher (set_ema(0.999)).
Prints one JSON line:
  sup_step_ms      a supervised training step (CUDA events, median), the teacher's EMA included; sup_step_no_teacher_ms
                   the same step before the teacher exists
  pl_ms            slimipl.pseudo_labels: the teacher's eval forward and CTC path, the copy to the host, the text round trip
                   (path -> letters -> words -> targets) and the copy back (host clock around a synchronised call, median)
  hard_step_ms     pl_ms plus the training step on those PLs (host clock, median).  The model has taken only the
                   steps timed before, so its PLs can be longer than a trained model's; they are capped at the workload's
                   60 tokens, so that the CTC step costs what it costs on real PLs (pl_tokens: the mean length before the
                   cap)
  soft_step_ms     slimipl.soft_targets (the teacher's eval forward) plus Trainer.step_soft (host clock, median)
  step_soft_ms     Trainer.step_soft alone (CUDA events, median)
  soft_loss_kernel w2l_soft_label_loss alone at rows = B T', N = 10 000 (CUDA events over 50 calls): time, the bytes it
                   must move (student and teacher read once, the gradient written once: 12 bytes per element) over that
                   time, and that rate over the H100 SXM's 3.35 TB/s HBM3 (data sheet)
  ema_ms           w2l_ema_update over the TDS arena and over the conv_glu LibriSpeech arena (CUDA events over 50 calls),
                   12 bytes per parameter, and the same rates
and the card's name, power limit and max SM clock, read in the same process.  Needs a CUDA device.

  python scripts/bench_slimipl.py [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12  # bytes/s, H100 SXM data sheet


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def events(fn, steps, warmup):
    import torch

    for _ in range(warmup):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    t = sorted(a.elapsed_time(b) for a, b in ev)
    return t[len(t) // 2]


def host(fn, steps, warmup):
    import torch

    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append(1e3 * (time.perf_counter() - t0))
    t.sort()
    return t[len(t) // 2]


def tokens_text(n):
    """n tokens: | ' a..z, then two- and three-letter strings (a word-piece-sized dictionary)"""
    import itertools
    import string

    toks = ["|", "'"] + list(string.ascii_lowercase)
    for k in (2, 3):
        for t in itertools.product(string.ascii_lowercase, repeat=k):
            if len(toks) == n:
                return "\n".join(toks) + "\n"
            toks.append("".join(t))
    return "\n".join(toks[:n]) + "\n"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()

    import numpy as np
    import torch

    from wav2letter_b200 import archs, capi
    from wav2letter_b200.slimipl import pseudo_labels, soft_targets
    from wav2letter_b200.text import TextPipeline
    from wav2letter_b200.trainer import Trainer

    if not torch.cuda.is_available():
        sys.exit("bench_slimipl.py needs a CUDA device")
    B, T, F, N, L = 16, 1200, 80, 10000, 60
    rng = np.random.default_rng(0)
    tr = Trainer(archs.seq2seq_tds(True), F, N, "ctc", "none", lr=0.05, maxgradnorm=15.0, precision="f32")
    text = TextPipeline(tokens_text(N - 1), "", "ctc", 0, "", False, "|")
    assert text.num_classes == N
    feat = torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32)).cuda()
    y = rng.integers(0, N - 1, (B, L)).astype(np.int32)
    for b, n in enumerate(rng.integers(L // 2, L + 1, B)):
        y[b, n:] = -1
    tgt = torch.from_numpy(y).cuda()
    out = {"card": card(), "workload": f"TDS+CTC B={B} T={T} F={F} N={N} f32, teacher decay 0.999"}

    out["sup_step_no_teacher_ms"] = events(lambda: tr.step(feat, tgt), args.steps, args.warmup)
    tr.set_ema(0.999)
    out["sup_step_ms"] = events(lambda: tr.step(feat, tgt), args.steps, args.warmup)
    out["pl_ms"] = host(lambda: pseudo_labels(tr, text, feat), args.steps, args.warmup)
    _, sizes, _ = pseudo_labels(tr, text, feat)
    out["pl_tokens"] = float(sizes.float().mean())

    def hard():
        t, _, _ = pseudo_labels(tr, text, feat)
        t = t[:, :L].contiguous()
        tr.step(feat, t)

    out["hard_step_ms"] = host(hard, args.steps, args.warmup)
    out["soft_step_ms"] = host(lambda: tr.step_soft(feat, soft_targets(tr, feat)), args.steps, args.warmup)
    teacher = soft_targets(tr, feat)
    out["step_soft_ms"] = events(lambda: tr.step_soft(feat, teacher), args.steps, args.warmup)
    assert tr.skipped_steps() == 0

    student = tr.forward(feat)
    rows = student.shape[0] * student.shape[1]
    d = torch.empty_like(student)
    ms = events(lambda: capi.soft_label_loss(student, teacher, 1.0, d_student=d), 50, 5)
    nbytes = 12 * rows * N
    out["soft_loss_kernel"] = {"rows": rows, "N": N, "ms": ms, "bytes": nbytes, "GBps": nbytes / ms / 1e6, "of_hbm_peak": nbytes / (ms * 1e-3) / HBM_PEAK}

    out["ema"] = {}
    glu = Trainer(archs.conv_glu_librispeech(), 40, 30, "asg", "none", precision="f32")
    for name, t in (("tds", tr), ("conv_glu", glu)):
        n = t.num_params(0)
        e = torch.zeros(n, dtype=torch.float32, device="cuda")
        p = t.get_flat(0)
        ms = events(lambda: capi.ema_update(e, p, 0.999), 50, 5)
        out["ema"][name] = {"params": n, "ms": ms, "GBps": 12 * n / ms / 1e6, "of_hbm_peak": 12 * n / (ms * 1e-3) / HBM_PEAK}
    glu.close()
    tr.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
