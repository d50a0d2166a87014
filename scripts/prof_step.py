"""Per-kernel breakdown of one train step of a bench.py workload (default tds_ctc, f32), everything on one stream.

The trainer is built from bench.WORKLOADS with the gradient stream off, so the traced launches run one after another
and each kernel's share is its own.  After warm-up, one step runs under capi.trace (a CUDA event after every launch);
the script prints the card, every kernel's launches, ms and share of the traced step, and the time-convolution
kernels summed.  Usage: python scripts/prof_step.py [workload] [precision]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from wav2letter_b200 import capi  # noqa: E402
from wav2letter_b200.trainer import Trainer  # noqa: E402

CONV_PREFIXES = ("conv_mma_", "conv_time_", "conv_wgrad_", "conv_arrange_")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def main():
    wl = sys.argv[1] if len(sys.argv) > 1 else "tds_ctc"
    cfg = bench.WORKLOADS[wl]
    prec = sys.argv[2] if len(sys.argv) > 2 else cfg["precision"]
    tr = Trainer(cfg["arch"], cfg["F"], cfg["N"], cfg["crit"], cfg["scale_mode"], transdiag=cfg["transdiag"], lr=cfg["lr"],
                 lrcrit=cfg["lrcrit"], momentum=cfg["momentum"], maxgradnorm=cfg["maxgradnorm"], precision=prec)
    tr.set_grad_stream(False)
    rng = np.random.default_rng(1234)
    sets = []
    for _ in range(4):
        f, y = bench.make_train_inputs(rng, cfg)
        sets.append((torch.from_numpy(f).cuda(), torch.from_numpy(y).cuda()))
    for i in range(6):
        tr.step(*sets[i % 4], True)
    torch.cuda.synchronize()
    agg = capi.trace(lambda: tr.step(*sets[0], True))
    torch.cuda.synchronize()
    total = sum(v[1] for v in agg.values()) or 1.0
    conv = {k: v for k, v in agg.items() if k.startswith(CONV_PREFIXES)}
    conv_ms = sum(v[1] for v in conv.values())
    print(f"card: {card()}")
    print(f"workload {wl}, precision {prec}, gradient stream off: traced step {total:.3f} ms, {sum(v[0] for v in agg.values())} launches")
    print(f"{'kernel':60s} {'launches':>8s} {'ms':>9s} {'share':>7s}")
    for k, (n, ms) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"{k:60s} {n:8d} {ms:9.3f} {100 * ms / total:6.1f}%")
    print(f"{'time convolution (' + ', '.join(sorted(conv)) + ')':60s} {sum(v[0] for v in conv.values()):8d} {conv_ms:9.3f} "
          f"{100 * conv_ms / total:6.1f}%")
    print(json.dumps({"workload": wl, "precision": prec, "traced_ms": total, "conv_ms": conv_ms,
                      "kernels": {k: {"launches": n, "ms": ms} for k, (n, ms) in agg.items()}}))
    tr.close()


if __name__ == "__main__":
    main()
