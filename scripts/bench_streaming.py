"""Throughput of the streaming acoustic model (wav2letter_b200/streaming.py) on the BASELINE streaming arch
(recipes/streaming_convnets/librispeech/am_500ms_future_context.arch, configs[3]).

For each precision and each count of concurrent streams, every stream is fed 500 ms chunks (50 feature frames at a
10 ms stride) in one `run` call per chunk, after warm-up calls.  Prints one JSON line per case:
  run_ms_device        device time per run call (CUDA events around each call, median; GEMM profiling off)
  audio_s_per_s        audio seconds processed per wall second (host clock around the same calls, synchronised)
  gemm_tflops          2*M*N*K of the call's GEMM launches over their event-timed duration, measured in a second loop
                       of calls; M is the padded batch's rows (streams x output frames of the layer, the shape
                       arithmetic of bench.py's arch_gemm_flops)
  state_bytes_per_stream
and the card's name and power limit, read in the same process.  Needs a CUDA device; there is no CPU path.

  python scripts/bench_streaming.py [--labels 10000] [--streams 1 64 512] [--precisions bf16 f32] [--calls 40]

--audio feeds raw audio instead: every stream gets 500 ms chunks (8000 samples at 16 kHz) through the MFSC front end
(StreamingFeatures, 80 filters, left_ctx 300) and its features go to the acoustic model in the same iteration.  Per
case it prints the device ms per call (median of event pairs) of the front end alone, of front end + AM, and of the AM
fed precomputed features, measured in alternating rounds in the same process, and the audio seconds per wall second of
front end + AM.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gemm_shapes(arch_text, n_feat, n_label, rows_per_conv):
    """(M, N, K) of every GEMM of one call, in launch order; rows_per_conv: padded rows after each convolution"""
    shapes, c, rows = [], 0, 0
    for line in arch_text.splitlines():
        p = line.replace("NFEAT", str(n_feat)).replace("NLABEL", str(n_label)).split()
        if not p:
            continue
        if p[0] in ("C2", "TDS"):
            rows = rows_per_conv[c]
            c += 1
        if p[0] == "TDS" and rows:
            d = int(p[1]) * int(p[3])
            inner = int(p[5]) if len(p) > 5 and int(p[5]) > 0 else d
            shapes += [(rows, inner, d), (rows, d, inner)]
        elif p[0] == "L" and rows:
            shapes.append((rows, int(p[2]), int(p[1])))
    return shapes


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--labels", type=int, default=10000)
    ap.add_argument("--streams", type=int, nargs="+", default=[1, 64, 512])
    ap.add_argument("--precisions", nargs="+", default=["bf16", "f32"])
    ap.add_argument("--chunk", type=int, default=50)
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--audio", action="store_true", help="raw 16 kHz audio through the streaming MFSC front end")
    ap.add_argument("--rounds", type=int, default=3, help="--audio: alternating rounds of the three variants")
    args = ap.parse_args()

    from wav2letter_b200 import archs, capi, streaming

    arch = archs.streaming_tds()
    # the frame arithmetic first: it runs on the host, so a machine without a device gets this far
    specs, frames, _ = streaming.plan(arch, 80, args.labels, [args.chunk] * (args.warmup + args.calls), finish=False)
    steady = frames[-1]
    shapes = gemm_shapes(arch, 80, args.labels, [int(f) for f in steady])
    flops_per_stream = sum(2 * m * n * k for m, n, k in shapes)
    print(json.dumps({"arch": "streaming_tds", "convolutions": len(specs), "steady_frames_per_conv": [int(f) for f in steady],
                      "gemm_flops_per_stream_per_call": flops_per_stream}), flush=True)

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_streaming: no CUDA device; the streaming runtime runs on the GPU only")
    from wav2letter_b200.trainer import Trainer

    dev = card()
    if args.audio:
        return audio_bench(args, arch, dev)
    for precision in args.precisions:
        tr = Trainer(arch, 80, args.labels, "ctc", "none", precision=precision)
        for S in args.streams:
            am = streaming.StreamingAM(tr, S, max_chunk=args.chunk, precision=precision)
            slots = list(range(S))
            am.start(slots)
            g = torch.Generator(device="cuda").manual_seed(S)
            x = torch.randn((S, 1, 80, args.chunk), device="cuda", generator=g)
            for _ in range(args.warmup):
                am.run(slots, x)
            torch.cuda.synchronize()
            # end to end with profiling off: device time per call (events around each call) and the wall clock
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.calls)]
            t0 = time.perf_counter()
            for a, b in ev:
                a.record()
                am.run(slots, x)
                b.record()
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            # then the GEMM launches alone, in a separate loop with an event pair around each
            prof = capi.ProfileList(1, len(shapes) * args.calls + 8)
            prof.arm()
            for _ in range(args.calls):
                am.run(slots, x)
            torch.cuda.synchronize()
            used = prof.disarm()
            call_ms = sorted(a.elapsed_time(b) for a, b in ev)
            gemm_ms = sum(prof.times_ms(used))
            gemm_flops = flops_per_stream * S * args.calls * used / max(1, len(shapes) * args.calls)
            print(json.dumps({
                "precision": precision, "streams": S, "chunk_frames": args.chunk, "labels": args.labels, "calls": args.calls,
                "run_ms_device": round(call_ms[len(call_ms) // 2], 4), "run_ms_device_min": round(call_ms[0], 4),
                "audio_s_per_s": round(S * args.calls * args.chunk * 0.01 / wall, 1),
                "gemm_tflops": round(gemm_flops / (gemm_ms * 1e-3) / 1e12, 2) if gemm_ms > 0 else None,
                "gemm_launches_timed": used, "gemm_ms_per_call": round(gemm_ms / args.calls, 4),
                "state_bytes_per_stream": am.state_bytes, "card": dev}), flush=True)
            am.close()
        tr.close()


def audio_bench(args, arch, dev):
    import torch

    from wav2letter_b200 import streaming
    from wav2letter_b200.trainer import Trainer

    samples = args.chunk * 160  # 10 ms stride at 16 kHz
    for precision in args.precisions:
        tr = Trainer(arch, 80, args.labels, "ctc", "none", precision=precision)
        for S in args.streams:
            fe = streaming.StreamingFeatures(S, samples)
            am = streaming.StreamingAM(tr, S, max_chunk=fe.max_frames_out, precision=precision)
            slots = list(range(S))
            fe.start(slots)
            am.start(slots)
            g = torch.Generator(device="cuda").manual_seed(S)
            audio = (torch.randn((S, samples), device="cuda", generator=g) * 1000).contiguous()
            x = torch.randn((S, 1, 80, args.chunk), device="cuda", generator=g)

            def front():
                fe.run(slots, audio)

            def both():
                f, frames = fe.run(slots, audio)
                am.run(slots, f, frames)

            def model():
                am.run(slots, x)

            variants = {"frontend": front, "frontend_am": both, "am_features": model}
            for fn in variants.values():  # warm every shape
                for _ in range(args.warmup):
                    fn()
            torch.cuda.synchronize()
            times = {k: [] for k in variants}
            walls = []
            for _ in range(args.rounds):
                for name, fn in variants.items():
                    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.calls)]
                    t0 = time.perf_counter()
                    for a, b in ev:
                        a.record()
                        fn()
                        b.record()
                    torch.cuda.synchronize()
                    if name == "frontend_am":
                        walls.append(time.perf_counter() - t0)
                    times[name] += [a.elapsed_time(b) for a, b in ev]
            med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
            print(json.dumps({
                "precision": precision, "streams": S, "chunk_samples": samples, "labels": args.labels, "calls": args.calls, "rounds": args.rounds,
                "frontend_ms_device": round(med["frontend"], 4), "frontend_am_ms_device": round(med["frontend_am"], 4),
                "am_features_ms_device": round(med["am_features"], 4),
                "frontend_share_of_am": round(med["frontend"] / med["am_features"], 4),
                "audio_s_per_s": round(S * args.calls * samples / 16000 / min(walls), 1),
                "frontend_state_bytes_per_stream": fe.state_bytes, "card": dev}), flush=True)
            am.close()
            fe.close()
        tr.close()


if __name__ == "__main__":
    main()
