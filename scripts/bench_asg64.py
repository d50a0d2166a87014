"""The 64-wide criterion calls and the TIMIT phone recipe's train step.

1. Fused ASG forward + backward and FCC Viterbi at T = 1500, B = 64 (L = 250, target_sz_sqrt): N = 30 through both
   calls, then N = 39 (the folded TIMIT phone set) and N = 61 through the 64-wide calls.  CUDA events over 20 launches
   after 3 warm-up launches, 4 rotating input sets.
2. One train step of recipes/learnable_frontend/am_baseline_conv_relu.arch (7 x C2 1000 + PReLU + dropout 0.7, ASG over
   39 tokens, the cfg's lr / lrcrit / momentum / maxgradnorm): B = 16, T = 300 (about 3 s of TIMIT audio), in f32, tf32
   and bf16, 10 steps after 3 warm-up steps.  The criterion's share is the 64-wide ASG call at the step's emission shape
   timed the same way, over the step time.
Prints the card's name, power limit and maximum SM clock first, then one JSON line per point with the SM clock read
right after its timed loop."""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from wav2letter_b200 import archs, capi  # noqa: E402
from wav2letter_b200.trainer import Trainer  # noqa: E402


def smi(fields):
    return subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()


def timed(fn, n=20, warm=3):
    for i in range(warm):
        fn(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, smi("clocks.sm")


def asg_point(B, T, N, L, wide, sets=4, seed=0):
    rng = np.random.default_rng(seed)
    data = []
    for _ in range(sets):
        e = (rng.normal(0, 1, (B, T, N)) * 3).astype(np.float32)
        y = rng.integers(0, N, (B, L)).astype(np.int32)
        data.append((torch.from_numpy(e).cuda(), torch.from_numpy(y).cuda()))
    trans = torch.from_numpy((4 * np.eye(N) + rng.normal(0, 0.1, (N, N))).astype(np.float32)).cuda()
    asg = capi.asg64_forward_backward if wide else capi.asg_forward_backward
    ws_size = capi.lib.w2l_asg64_workspace_size if wide else capi.lib.w2l_asg_workspace_size
    out = (torch.empty(B, device="cuda"), torch.empty((B, T, N), device="cuda"), torch.empty((N, N), device="cuda"))
    ws = torch.empty(ws_size(B, T, N, L), dtype=torch.uint8, device="cuda")
    return data, trans, lambda i: asg(data[i % sets][0], data[i % sets][1], trans, "target_sz_sqrt", out=out, ws=ws)


def main():
    print(smi("name,power.limit,clocks.max.sm"))
    B, T, L = 64, 1500, 250
    for N, wide in ((30, False), (30, True), (39, True), (61, True)):
        data, trans, step = asg_point(B, T, N, L, wide, seed=N)
        vit = capi.fcc_viterbi64 if wide else capi.fcc_viterbi
        asg_ms, clk = timed(step)
        vit_ms, _ = timed(lambda i: vit(data[i % 4][0], trans))
        print(json.dumps({"N": N, "call": "64" if wide else "32", "B": B, "T": T, "L": L, "asg_fwd_bwd_ms": round(asg_ms, 3),
                          "fcc_viterbi_ms": round(vit_ms, 3), "sm_clock": clk}))
    # the TIMIT train step
    B, T, L, N, F = 16, 300, 40, 39, 40
    rng = np.random.default_rng(1)
    feat = torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32)).cuda()
    tgt = torch.from_numpy(rng.integers(0, N, (B, L)).astype(np.int32)).cuda()
    for precision in ("f32", "tf32", "bf16"):
        tr = Trainer(archs.learnable_frontend_timit(), F, N, "asg", "target_sz_sqrt", lr=0.1, lrcrit=0.1, momentum=0.5,
                     maxgradnorm=1.0, precision=precision)
        Tout = tr.forward(feat).shape[1]
        step_ms, clk = timed(lambda i: tr.step(feat, tgt, True, float(B)), n=10)
        tr.close()
        _, _, crit = asg_point(B, Tout, N, L, True, seed=2)
        crit_ms, _ = timed(crit)
        print(json.dumps({"workload": "learnable_frontend_timit", "precision": precision, "B": B, "T": T, "N": N,
                          "step_ms": round(step_ms, 3), "asg64_ms": round(crit_ms, 3),
                          "criterion_share": round(crit_ms / step_ms, 4), "sm_clock": clk}))
    capi.set_precision("tf32")


if __name__ == "__main__":
    main()
