"""Cost of the criterion's path in the streaming acoustic model (StreamingAM.run(..., path=True), w2l_stream_run_path)
on the BASELINE streaming arch (streaming_tds), at 512 streams of 500 ms chunks (50 feature frames) in bf16.

For CTC over 10 000 word pieces and ASG over 30 letters it times, in alternating rounds in one process (CUDA events
around each call, median):
  run_ms              the call without a path (w2l_stream_run, emissions copied out)
  path_emis_ms        the call with the path and the emissions
  path_only_ms        the call with the path alone (emissions = NULL: no emission copy)
and what a caller must copy back to the host per call to get tokens:
  emission_bytes      streams x output frames x N x 4 (the emissions, to decode them elsewhere)
  path_bytes          streams x (3 + entries committed in the call) x 4 (path_info and the committed entries; the
                      entries are those of the last timed call)
with the card's name and power limit, read in the same process.  Needs a CUDA device.

  python scripts/bench_streaming_path.py [--streams 512] [--chunk 50] [--calls 40] [--rounds 3]
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
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=512)
    ap.add_argument("--chunk", type=int, default=50)
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--precision", default="bf16")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_streaming_path: no CUDA device; the streaming runtime runs on the GPU only")
    from wav2letter_b200 import archs, streaming
    from wav2letter_b200.trainer import Trainer

    dev = card()
    arch = archs.streaming_tds()
    S = args.streams
    slots = list(range(S))
    for crit, N in (("ctc", 10000), ("asg", 30)):
        tr = Trainer(arch, 80, N, crit, "none", precision=args.precision)
        am = streaming.StreamingAM(tr, S, max_chunk=args.chunk, precision=args.precision)
        am.start(slots)
        g = torch.Generator(device="cuda").manual_seed(S)
        x = torch.randn((S, 1, 80, args.chunk), device="cuda", generator=g)
        last = {}

        def plain():
            last["fo"] = am.run(slots, x)[1]

        def with_emissions():
            am.run(slots, x, path=True)

        def path_only():
            last["info"] = am.run(slots, x, path=True, emissions=False)[3]

        variants = {"run_ms": plain, "path_emis_ms": with_emissions, "path_only_ms": path_only}
        for fn in variants.values():
            for _ in range(args.warmup):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in variants}
        for _ in range(args.rounds):
            for name, fn in variants.items():
                ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.calls)]
                for a, b in ev:
                    a.record()
                    fn()
                    b.record()
                torch.cuda.synchronize()
                times[name] += [a.elapsed_time(b) for a, b in ev]
        med = {k: round(sorted(v)[len(v) // 2], 4) for k, v in times.items()}
        frames = max(last["fo"])
        committed = int(last["info"][:, 1].sum())
        print(json.dumps({
            "criterion": crit, "labels": N, "streams": S, "chunk_frames": args.chunk, "precision": args.precision, "calls": args.calls,
            "rounds": args.rounds, **med, "output_frames_per_stream": frames, "emission_bytes": S * frames * N * 4,
            "path_bytes": (3 * S + committed) * 4, "path_state_bytes_per_stream": am.state_bytes, "card": dev}), flush=True)
        am.close()
        tr.close()


if __name__ == "__main__":
    main()
