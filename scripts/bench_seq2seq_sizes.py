"""The Seq2Seq criterion on padded batches: the seq2seq_tds training step, greedy decode and K = 4 beam search with and
without per-utterance sizes, in one process, alternating the variants of each call so that drift hits them alike.

Workload (fp32-accurate precision, the recipe's TDS encoder archs.seq2seq_tds(ctc_head=False), 80 filterbanks, B = 16
utterances padded to 1200 frames -> T' = 150, N = 10002 classes with eos and pad, U = 61, H = 512, the trainer's random
initialisation; lr = 0 so every repeat runs the same model):
  step      unsized; sized at full length (every duration 1200, every target size U); sized with durations spread
            from 900 to 1200 frames and target sizes from 41 to 61
  decode    greedy decode (maxdecoderoutputlen 150) of the spread batch, unsized and sized
  beam      the K = 4 beam search (maxlen 150) of the spread batch, unsized and sized
Prints one JSON line per call and variant: ms (median of --rounds rounds, each the CUDA-event time of one call after
warm-up), the spread of the rounds (min, max), and the card's name, power limit and max SM clock read in the same
process.  Needs a CUDA device.

  python scripts/bench_seq2seq_sizes.py [--rounds 15] [--warmup 3]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_seq2seq import card  # noqa: E402


def alternate(variants, rounds, warmup):
    """{name: [ms of each round]}: every round calls each variant once, in order, between CUDA events"""
    import torch

    for _ in range(warmup):
        for fn in variants.values():
            fn()
    times = {k: [] for k in variants}
    for _ in range(rounds):
        for k, fn in variants.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b))
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import numpy as np
    import torch

    from wav2letter_b200 import archs
    from wav2letter_b200.trainer import Trainer

    assert torch.cuda.is_available(), "bench_seq2seq_sizes needs a CUDA device"
    info = card()
    B, T, F, N, U, H, K, maxlen = 16, 1200, 80, 10002, 61, 512, 4, 150
    rng = np.random.default_rng(0)
    d = np.linspace(900, 1200, B).round().astype(int)[::-1].copy()
    n = np.linspace(40, 60, B).round().astype(int)[::-1].copy()
    feat = rng.standard_normal((B, 1, F, T), dtype=np.float32)
    for b in range(B):
        feat[b, :, :, d[b]:] = 0
    feat = torch.from_numpy(feat).cuda()
    y = np.full((B, U), N - 1, np.int32)
    for b in range(B):
        y[b, :n[b]] = rng.integers(0, N - 2, n[b])
        y[b, n[b]] = N - 2
    tgt = torch.from_numpy(y).cuda()
    dev = lambda v: torch.tensor([int(x) for x in v], dtype=torch.int32, device="cuda")  # noqa: E731
    full_d, full_u, spread_d, spread_u = dev([T] * B), dev([U] * B), dev(d), dev(n + 1)
    arch = archs.seq2seq_tds(ctc_head=False).replace("L 1440 1024", f"L 1440 {2 * H}")
    tr = Trainer(arch, F, N, "seq2seq", lr=0.0, lrcrit=0.0, precision="f32",
                 seq2seq=dict(hidden=H, eos=N - 2, pad=N - 1, maxdecoderoutputlen=maxlen))
    calls = {
        "step": {
            "unsized": lambda: tr.step(feat, tgt),
            "sized_full": lambda: tr.step(feat, tgt, input_sizes=full_d, target_sizes=full_u),
            "sized_spread": lambda: tr.step(feat, tgt, input_sizes=spread_d, target_sizes=spread_u),
        },
        "greedy_decode": {"unsized": lambda: tr.decode(feat), "sized_spread": lambda: tr.decode(feat, input_sizes=spread_d)},
        "beam_search_k4": {"unsized": lambda: tr.beam_search(feat, K), "sized_spread": lambda: tr.beam_search(feat, K, input_sizes=spread_d)},
    }
    for call, variants in calls.items():
        rounds = args.rounds if call == "step" else max(3, args.rounds // 3)
        for k, t in alternate(variants, rounds, args.warmup if call == "step" else 1).items():
            t = sorted(t)
            print(json.dumps({"call": call, "variant": k, "B": B, "T": T, "ms": round(t[len(t) // 2], 3), "min_ms": round(t[0], 3),
                              "max_ms": round(t[-1], 3), "rounds": len(t), "card": info}), flush=True)


if __name__ == "__main__":
    main()
