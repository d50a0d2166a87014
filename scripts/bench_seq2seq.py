"""The seq2seq_tds recipe's training step with the Seq2Seq criterion, beside TDS+CTC on the same batch, in one process.

Workloads (fp32-accurate precision, B = 16 utterances of 1200 frames, 80 filterbanks, the recipe's TDS encoder
archs.seq2seq_tds(ctc_head=False), N = 10002 classes with eos and pad, U = 61 decoder steps including eos, H = 512):
  s2s_r1s1   the seq2seq_tds recipe's decoder: 1 attention round, 1 GRU layer
  s2s_r2s3   the sota/2019 tds_s2s decoder: 2 rounds of 3 GRU layers, decoder dropout 0.1
  s2s_h1024  the same decoder at --encoderdim=1024 (the librivox tds_s2s setting), the encoder's last layer widened to
             `L 1440 2048`
  ctc        archs.seq2seq_tds(ctc_head=True) with CTC over 10000 tokens (bench.py's configs[1]), same batch
Prints one JSON line per workload:
  step_ms              median device time of a training step (CUDA events around each step, after warm-up)
  kernels_ms           one traced step (w2l_trace_*: an event after every launch): the Seq2Seq kernels' totals --
                       recurrence forward / backward (and us per decoder step per layer), attention, loss -- the GEMM
                       launches inside the criterion's forward (its input and output projections), the output
                       projection's forward GEMM alone, and all GEMM launches of the step
  criterion_fwd_ms     the traced criterion forward (embedding .. loss, contiguous in launch order)
  decode_ms            greedy decode of the batch at maxdecoderoutputlen = 120 (the encoder forward included; an
                       untrained model rarely emits eos, so this is close to the full 120 steps)
and the card's name, power limit and max SM clock, read in the same process.  Needs a CUDA device.

  python scripts/bench_seq2seq.py [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def timed(fn, steps, warmup):
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


def breakdown(fn, U, layers):
    from wav2letter_b200 import capi

    capi.trace(fn, capacity=16384)
    seq = capi.trace_list()
    names = [n for n, _ in seq]
    tot = lambda pred, lst=seq: sum(ms for n, ms in lst if pred(n))  # noqa: E731
    is_gemm = lambda n: "gemm" in n  # noqa: E731
    lo, hi = names.index("seq2seq_embed_fwd_kernel"), names.index("seq2seq_loss_sum_kernel")
    fwd = seq[lo:hi + 1]
    last_attn = max(i for i, n in enumerate(names[:hi + 1]) if n == "seq2seq_attn_fwd_kernel")
    rec_f, rec_b = tot(lambda n: n == "seq2seq_gru_fwd_kernel"), tot(lambda n: n == "seq2seq_gru_bwd_kernel")
    return {
        "recurrence_fwd_ms": round(rec_f, 4), "recurrence_bwd_ms": round(rec_b, 4),
        "recurrence_fwd_us_per_step_layer": round(1000 * rec_f / (U * layers), 3),
        "recurrence_bwd_us_per_step_layer": round(1000 * rec_b / (U * layers), 3),
        "attention_ms": round(tot(lambda n: n.startswith("seq2seq_attn")), 4),
        "loss_ms": round(tot(lambda n: n.startswith("seq2seq_loss")), 4),
        "embedding_ms": round(tot(lambda n: n.startswith("seq2seq_embed")), 4),
        "criterion_fwd_gemm_ms": round(tot(is_gemm, fwd), 4),
        "output_gemm_fwd_ms": round(tot(is_gemm, seq[last_attn:hi + 1]), 4),
        "step_gemm_ms": round(tot(is_gemm), 4),
    }, round(sum(ms for _, ms in fwd), 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()

    import numpy as np
    import torch

    from wav2letter_b200 import archs
    from wav2letter_b200.trainer import Trainer

    assert torch.cuda.is_available(), "bench_seq2seq needs a CUDA device"
    B, T, F, N, U, H = 16, 1200, 80, 10002, 61, 512
    rng = np.random.default_rng(0)
    feat = torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32)).cuda()
    y = np.full((B, U), N - 1, np.int32)
    for b in range(B):
        n = U - 1 - (b % 8)
        y[b, :n] = rng.integers(0, N - 2, n)
        y[b, n] = N - 2
    tgt = torch.from_numpy(y).cuda()
    info = card()
    ctc_y = torch.from_numpy(rng.integers(0, 9999, (B, U - 1)).astype(np.int32)).cuda()
    ctc = Trainer(archs.seq2seq_tds(ctc_head=True), F, 10000, "ctc", lr=0.01, precision="f32")
    print(json.dumps({"workload": "ctc", "step_ms": round(timed(lambda: ctc.step(feat, ctc_y), args.steps, args.warmup), 3), "card": info}), flush=True)
    del ctc
    for name, hidden, rounds, layers, p in (("s2s_r1s1", H, 1, 1, 0.0), ("s2s_r2s3", H, 2, 3, 0.1), ("s2s_h1024", 1024, 2, 3, 0.1)):
        arch = archs.seq2seq_tds(ctc_head=False).replace("L 1440 1024", f"L 1440 {2 * hidden}")
        tr = Trainer(arch, F, N, "seq2seq", lr=0.01, lrcrit=0.01, precision="f32",
                     seq2seq=dict(hidden=hidden, eos=N - 2, pad=N - 1, maxdecoderoutputlen=120, rounds=rounds, layers=layers, dropout=p))
        step = timed(lambda: tr.step(feat, tgt), args.steps, args.warmup)
        kern, crit_fwd = breakdown(lambda: tr.step(feat, tgt), U, rounds * layers)
        dec = timed(lambda: tr.decode(feat), max(3, args.steps // 4), 1)
        print(json.dumps({"workload": name, "step_ms": round(step, 3), "criterion_fwd_ms": crit_fwd, "kernels_ms": kern,
                          "decode_ms": round(dec, 3), "card": info}), flush=True)
        del tr


if __name__ == "__main__":
    main()
