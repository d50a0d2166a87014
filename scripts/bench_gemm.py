"""Time the train step's GEMM shapes for every tile width (w2l_gemm_set_tile) — calibration of the host heuristic."""
import os, sys, json
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import wav2letter_b200 as w
capi = w.capi

shapes = []
for M, C in [(9600, 800), (4800, 1120), (2400, 1440)]:
    shapes += [("fwd", M, C, C, False, False), ("dgrad", M, C, C, False, True), ("wgrad", C, C, M, True, True)]
shapes += [("head_fwd", 2400, 10000, 1440, False, False), ("head_dgrad", 2400, 1440, 10000, False, True),
           ("head_wgrad", 10000, 1440, 2400, True, True)]
nset = 4
out = {}
for name, M, N, K, a_mn, b_mn in shapes:
    As = [torch.randn((K, M) if a_mn else (M, K), device="cuda") for _ in range(nset)]
    Bs = [torch.randn((K, N) if b_mn else (N, K), device="cuda") for _ in range(nset)]
    C = torch.empty(M, N, device="cuda")
    row = {}
    for bn in (0, 128, 160, 224, 256):
        capi.gemm_set_tile(bn)
        for i in range(3):
            capi.gemm_tf32_ex(As[i % nset], Bs[i % nset], C, a_mn=a_mn, b_mn=b_mn)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 20
        e0.record()
        for i in range(n):
            capi.gemm_tf32_ex(As[i % nset], Bs[i % nset], C, a_mn=a_mn, b_mn=b_mn)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) / n * 1e3
        row[bn] = (round(us, 1), round(2.0 * M * N * K / us / 1e6, 1))
    capi.gemm_set_tile(0)
    out[f"{name} M={M} N={N} K={K}"] = row
    print(f"{name:11s} M={M:5d} N={N:5d} K={K:5d} " + "  ".join(f"bn{bn}: {v[0]:7.1f}us {v[1]:6.1f}TF" for bn, v in row.items()), flush=True)
json.dump(out, sys.stdout, indent=1)
