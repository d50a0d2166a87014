"""Throughput of MFSC featurisation (w2l_mfsc) on the GPU next to the NumPy reference's float32 path on the host cores.

Workload: one LibriSpeech-shaped batch — 16 utterances with log-normal lengths of mean 12.3 s, clipped to [0.5 s, 33 s],
16 kHz, 80 filters, 25 ms frames every 10 ms — featurised with per-utterance (left_ctx 0) and local (left_ctx 300)
normalisation.  GPU: CUDA events around `--iters` calls after `--warmup`; a traced call splits the time per kernel.
CPU: tests/features_reference.py in float32 (BLAS GEMM for the folded DFT), one utterance per worker thread.
Prints one JSON line; writes nothing.

    python scripts/bench_features.py [--iters 50] [--warmup 5] [--threads N]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import features_reference as R  # noqa: E402

FS = 16000
STEP_FRAMES = 16 * 1200  # frames of the README's train step (B = 16 x T = 1200)


def librispeech_lengths(B, seed):
    rng = np.random.default_rng(seed)
    sigma = 0.6
    s = rng.lognormal(np.log(12.3) - sigma * sigma / 2, sigma, B)
    return [int(v * FS) for v in np.clip(s, 0.5, 33.0)]


def synth(n, rng):
    f0 = np.repeat(rng.uniform(90, 280, n // 1600 + 1), 1600)[:n]
    phase = np.cumsum(2 * np.pi * f0 / FS)
    x = sum(rng.uniform(0.2, 1.0) / h * np.sin(h * phase) for h in range(1, 9))
    return 2000.0 * x + rng.normal(0, 30.0, n)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [v.strip() for v in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # pragma: no cover
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"not read ({e})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--threads", type=int, default=os.cpu_count())
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_features.py needs a CUDA device")

    from wav2letter_b200 import capi
    from wav2letter_b200.features import mfsc

    lengths = librispeech_lengths(args.batch, args.seed)
    rng = np.random.default_rng(args.seed + 1)
    audio = np.zeros((args.batch, max(lengths)), dtype=np.float32)
    for b, n in enumerate(lengths):
        audio[b, :n] = synth(n, rng)
    frames = sum(R.num_frames(n, FS, 25, 10) for n in lengths)
    dev = torch.from_numpy(audio).cuda()
    out = {"workload": {"utterances": args.batch, "seconds": round(sum(lengths) / FS, 2), "frames": frames,
                        "max_seconds": round(max(lengths) / FS, 2), "n_filters": 80, "frame_ms": 25, "stride_ms": 10},
           "gpu": gpu_info()}
    for left in (0, 300):
        for _ in range(args.warmup):
            mfsc(dev, lengths, left_ctx=left)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            mfsc(dev, lengths, left_ctx=left)
        b.record()
        b.synchronize()
        ms = a.elapsed_time(b) / args.iters
        traced = capi.trace(lambda: mfsc(dev, lengths, left_ctx=left))
        out[f"gpu_left_ctx_{left}"] = {
            "ms_per_batch": round(ms, 4), "frames_per_s": round(frames / ms * 1e3),
            "ms_per_train_step_batch": round(STEP_FRAMES / (frames / ms), 4),
            "kernels_ms": {k: round(v[1], 4) for k, v in sorted(traced.items())}}

    # CPU baseline: the reference's float32 path, one utterance per worker
    p = R.Params(FS, 25, 10, 80, np.float32)
    utts = [audio[b, :n] for b, n in enumerate(lengths)]
    R.mfsc_utterance(p, utts[0][: 2 * FS])
    with ThreadPoolExecutor(args.threads) as pool:
        t0 = time.perf_counter()
        list(pool.map(lambda x: R.mfsc_utterance(p, x), utts))
        cpu_s = time.perf_counter() - t0
    out["cpu_numpy_f32"] = {"threads": args.threads, "host_cpus": os.cpu_count(), "s_per_batch": round(cpu_s, 4),
                            "frames_per_s": round(frames / cpu_s)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
