"""The Seq2Seq criterion's beam search (Trainer.beam_search) beside the greedy decode of the same batch and beside B
single-utterance searches (the per-utterance loop local_prior_match's batchBeamSearch runs), in one process.

Shapes (fp32-accurate precision, the seq2seq_tds TDS encoder archs.seq2seq_tds(ctc_head=False) with its last layer
`L 1440 2H`, 80 filterbanks, 1200 frames -> T' = 150, the trainer's random initialisation):
  lpm          local_prior_match's proposal model: B = 2, K = 4 (--lpmBeamsz), H = 512, N = 5002, maxlen 150
  seq2seq_tds  the recipe's decoder: B = 16, K = 4, H = 512, N = 10002, maxlen 150
Prints one JSON line per shape and call: ms per call (median of CUDA-event pairs after warm-up, the encoder forward
included), the decoder steps one call ran (from a traced call: the step kernel's launches; an untrained model rarely
emits eos, so the searches run close to maxlen), and ms per step; then the card's name, power limit and max SM clock,
read in the same process.  Needs a CUDA device.

  python scripts/bench_seq2seq_beam.py [--calls 5] [--warmup 1]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_seq2seq import card, timed  # noqa: E402


def steps_of(fn, kernel):
    from wav2letter_b200 import capi

    got = capi.trace(fn, capacity=65536)
    return int(got[kernel][0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()

    import numpy as np
    import torch

    from wav2letter_b200 import archs
    from wav2letter_b200.trainer import Trainer

    assert torch.cuda.is_available(), "bench_seq2seq_beam needs a CUDA device"
    info = card()
    T, F, H, K, maxlen = 1200, 80, 512, 4, 150
    for name, B, N in (("lpm", 2, 5002), ("seq2seq_tds", 16, 10002)):
        rng = np.random.default_rng(0)
        feat = torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32)).cuda()
        arch = archs.seq2seq_tds(ctc_head=False).replace("L 1440 1024", f"L 1440 {2 * H}")
        tr = Trainer(arch, F, N, "seq2seq", lr=0.0, precision="f32", seq2seq=dict(hidden=H, eos=N - 2, pad=N - 1, maxdecoderoutputlen=maxlen))
        singles = [feat[b:b + 1].contiguous() for b in range(B)]
        calls = {
            "beam_search": (lambda: tr.beam_search(feat, K), "seq2seq_beam_topk_kernel"),
            "greedy_decode": (lambda: tr.decode(feat), "seq2seq_decode_step_kernel"),
            "single_utterance_beam_searches": (lambda: [tr.beam_search(x, K) for x in singles], "seq2seq_beam_topk_kernel"),
        }
        for call, (fn, kernel) in calls.items():
            ms = timed(fn, args.calls, args.warmup)
            steps = steps_of(fn, kernel)
            print(json.dumps({"shape": name, "B": B, "K": K, "H": H, "N": N, "maxlen": maxlen, "call": call, "ms": round(ms, 3), "steps": steps,
                              "ms_per_step": round(ms / steps, 4), "card": info}), flush=True)
        del tr


if __name__ == "__main__":
    main()
