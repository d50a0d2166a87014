"""Forward / stride-1 data gradient of the TDS time convolution: the wgmma kernel (path 3) against the mma.sync kernel
(path 2) on the shapes of the seq2seq_tds and streaming steps, with and without dropout.  Prints the timings as JSON."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from wav2letter_b200 import capi  # noqa: E402


def time_fwd(x, wt, bias, T, pl, p, path, iters=20):
    capi._check(capi.lib.w2l_conv_set_path(path))
    for _ in range(3):
        capi.conv_time_fwd(x, wt, bias, T, 1, pl, act=1, dropout_p=p, seed=5)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        capi.conv_time_fwd(x, wt, bias, T, 1, pl, act=1, dropout_p=p, seed=5)
    t1.record()
    torch.cuda.synchronize()
    capi._check(capi.lib.w2l_conv_set_path(0))
    return t0.elapsed_time(t1) / iters * 1e3


out = []
for (B, T, C, K, pl) in [(16, 600, 10, 21, 10), (16, 300, 14, 21, 10), (16, 150, 18, 21, 10), (8, 500, 15, 9, 7), (8, 250, 19, 9, 7),
                         (8, 125, 23, 11, 9), (8, 125, 27, 11, 10)]:
    x = torch.randn(B, T, C, 80, device="cuda")
    wt = torch.randn(C, C, K, device="cuda") * 0.1
    bias = torch.randn(C, device="cuda")
    rec = {"B": B, "T": T, "C": C, "K": K, "MB": round(2 * x.numel() * 4 / 1e6, 1)}
    for p in (0.0, 0.2):
        rec[f"wgmma_us_p{p}"] = round(time_fwd(x, wt, bias, T, pl, p, 3), 1)
        rec[f"mma_us_p{p}"] = round(time_fwd(x, wt, bias, T, pl, p, 2), 1)
    rec["wgmma_GBps"] = round(rec["MB"] * 1e3 / rec["wgmma_us_p0.2"], 1)
    rec["mma_GBps"] = round(rec["MB"] * 1e3 / rec["mma_us_p0.2"], 1)
    out.append(rec)
    print(json.dumps(rec), flush=True)
json.dump(out, sys.stdout, indent=1)
