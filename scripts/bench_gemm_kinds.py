"""Isolated timing of the wgmma GEMM in its three operand kinds on the 12 contraction shapes of the seq2seq_tds train
step (forward, data gradient, weight gradient of the FC layers of each stage + the 10 000-class head).  Inputs rotate
over enough buffers to exceed the 50 MB L2.  Prints one JSON record per shape (us and TFLOP/s per kind), then the list."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import wav2letter_b200 as w  # noqa: E402

SHAPES = [("stage1 fc", 9600, 800, 800), ("stage2 fc", 4800, 1120, 1120), ("stage3 fc", 2400, 1440, 1440), ("head", 2400, 10000, 1440)]


def time_one(kind, M, N, K, a_mn, b_mn, iters=20):
    dt = torch.bfloat16 if kind == "bf16" else torch.float32
    nbuf = max(2, int(200e6 // ((M * K + N * K) * (2 if kind == "bf16" else 4) + M * N * 4)) + 1)
    As = [torch.randn((K, M) if a_mn else (M, K), device="cuda").to(dt) for _ in range(nbuf)]
    Bs = [torch.randn((K, N) if b_mn else (N, K), device="cuda").to(dt) for _ in range(nbuf)]
    Cs = [torch.empty(M, N, device="cuda") for _ in range(nbuf)]
    for i in range(3):
        w.capi.gemm(As[i % nbuf], Bs[i % nbuf], kind, a_mn, b_mn, out=Cs[i % nbuf])
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(iters):
        w.capi.gemm(As[i % nbuf], Bs[i % nbuf], kind, a_mn, b_mn, out=Cs[i % nbuf])
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters * 1e3  # us


def main():
    out = []
    for name, rows, nout, nin in SHAPES:
        # forward Y[rows][nout] = X W^T; dgrad dX[rows][nin] = dY W; wgrad dW[nout][nin] = dY^T X
        for op, (M, N, K, a_mn, b_mn) in {"fwd": (rows, nout, nin, False, False), "dgrad": (rows, nin, nout, False, True),
                                          "wgrad": (nout, nin, rows, True, True)}.items():
            rec = {"shape": name, "op": op, "M": M, "N": N, "K": K}
            for kind in ("tf32", "f32x3", "bf16"):
                us = time_one(kind, M, N, K, a_mn, b_mn)
                rec[kind + "_us"] = round(us, 2)
                rec[kind + "_tflops"] = round(2.0 * M * N * K / us / 1e6, 1)
            out.append(rec)
            print(json.dumps(rec), flush=True)
    json.dump(out, sys.stdout, indent=1)


if __name__ == "__main__":
    main()
