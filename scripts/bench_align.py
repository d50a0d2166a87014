"""Forced-alignment timings on the GPU.

1. w2l_ctc_viterbi_target at B = 16, T' in {150, 400, 1500} output frames, N = 10 000 (the TDS + CTC word-piece set),
   L = T'/3: CUDA events around `--iters` calls after `--warmup`, and the median over `--iters` calls of the walk alone
   (ctc_align_kernel: forward recursion + backtrace; the rest of the call is the gather kernel).  The walk is T' dependent steps, so
   its time per frame (ns) is the figure to compare with the ASG chains.
2. Trainer.align against Trainer.forward on one 16 x 1200-frame batch of the seq2seq TDS + CTC model (bench.py's
   tds_ctc workload): the alignment's cost on top of the eval-mode forward it contains.
Prints one JSON line; writes nothing.

    python scripts/bench_align.py [--iters 20] [--warmup 3]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [v.strip() for v in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # pragma: no cover
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"not read ({e})"}


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_align.py needs a CUDA device")

    from wav2letter_b200 import archs, capi
    from wav2letter_b200.trainer import Trainer

    out = {"gpu": gpu_info()}
    rng = np.random.default_rng(0)
    B, N = 16, 10000
    for T in (150, 400, 1500):
        L = T // 3
        e = torch.from_numpy(rng.normal(0, 2, (B, T, N)).astype(np.float32)).cuda()
        y = torch.from_numpy(rng.integers(0, N - 1, (B, L)).astype(np.int32)).cuda()
        fn = lambda: capi.ctc_viterbi_target(e, y, return_state=True)
        ms = timed(fn, args.iters, args.warmup)
        # the walk alone: the library's event pair around each call's dominant kernel
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        capi.set_profile_events(a, b)
        walks = []
        for _ in range(args.iters):
            fn()
            b.synchronize()
            walks.append(a.elapsed_time(b))
        capi.set_profile_events(None)
        walk = float(np.median(walks))
        out[f"ctc_viterbi_T{T}"] = {"B": B, "T": T, "N": N, "L": L, "ms_per_call": round(ms, 4), "walk_ms": round(walk, 4),
                                    "walk_ns_per_frame": round(walk * 1e6 / T, 1)}
        del e

    tr = Trainer(archs.seq2seq_tds(True), 80, N, "ctc")
    Bt, Tt, L = 16, 1200, 60
    feat = torch.from_numpy(rng.normal(0, 1, (Bt, 1, 80, Tt)).astype(np.float32)).cuda()
    y = torch.from_numpy(rng.integers(0, N - 1, (Bt, L)).astype(np.int32)).cuda()
    fwd = timed(lambda: tr.forward(feat), args.iters, args.warmup)
    aln = timed(lambda: tr.align(feat, y), args.iters, args.warmup)
    _, idx = tr.align(feat, y)
    out["trainer_tds_ctc"] = {"B": Bt, "T": Tt, "T_out": int(idx.shape[1]), "N": N, "L": L, "time_stride": tr.time_stride(),
                              "forward_ms": round(fwd, 3), "align_ms": round(aln, 3), "align_over_forward_ms": round(aln - fwd, 3),
                              "aligned_utterances": int((idx[:, 0] >= 0).sum())}
    tr.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
