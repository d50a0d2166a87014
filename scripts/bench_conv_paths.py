"""Time the tensor-core time convolution (w2l_conv_time_{fwd,dgrad,wgrad}) at the shapes of the seq2seq_tds and
streaming_tds steps, in f32 (3xTF32) and tf32.

seq2seq_tds (B = 16, W = 80): the strided C2 convolutions 1->10, 10->14, 14->18 (kw 21, stride 2, T 1200/600/300; their
data gradient runs as two polyphase stride-1 launches) and the TDS convolutions C = 10/14/18 at T' = 600/300/150 (kw 21,
stride 1).  streaming_tds (B = 8): its TDS convolutions.  For each shape and direction the script prints µs per call,
algorithmic GB/s (read x + write y; read dy + write dx; read x + dy for the weight gradient) and TFLOP/s over the
padded MMA work the kernels issue (16-row M tiles, K padded to 8, three MMAs per product in f32).  The last record sums
one seq2seq step's convolutions: 14 forward, 13 data-gradient calls (15 launches) and 14 weight gradients.
Usage: python scripts/bench_conv_paths.py [out.json]"""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from wav2letter_b200 import capi  # noqa: E402

W = 80
# (name, B, T, Cin, Cout, K, stride, pad_left, calls per seq2seq step: fwd, dgrad, wgrad)
SHAPES = [("s2s C2 1->10", 16, 1200, 1, 10, 21, 2, 10, (1, 0, 1)),
          ("s2s C2 10->14", 16, 600, 10, 14, 21, 2, 10, (1, 1, 1)),
          ("s2s C2 14->18", 16, 300, 14, 18, 21, 2, 10, (1, 1, 1)),
          ("s2s TDS 10", 16, 600, 10, 10, 21, 1, 10, (2, 2, 2)),
          ("s2s TDS 14", 16, 300, 14, 14, 21, 1, 10, (3, 3, 3)),
          ("s2s TDS 18", 16, 150, 18, 18, 21, 1, 10, (6, 6, 6)),
          ("streaming TDS 15", 8, 500, 15, 15, 9, 1, 7, None),
          ("streaming TDS 19", 8, 250, 19, 19, 9, 1, 7, None),
          ("streaming TDS 23", 8, 125, 23, 23, 11, 1, 9, None),
          ("streaming TDS 27", 8, 125, 27, 27, 11, 1, 10, None)]


def tout_of(T, K, stride, pl):
    return (T + 2 * pl - K) // stride + 1  # symmetric padding, as the archs use


def mma_flops(B, frames, cout, kc, x3):
    """2 * (M padded to 16) * (K padded to 8) * W per output frame, x3 for 3xTF32"""
    return 2 * B * frames * 16 * ((cout + 15) // 16) * ((kc + 7) // 8 * 8) * W * (3 if x3 else 1)


def dgrad_flops(B, T, Tout, Cin, Cout, K, stride, pl, x3):
    if stride == 1:
        return mma_flops(B, T, Cin, K * Cout, x3)
    total = 0
    for p in range(stride):  # the polyphase split of w2l_conv_time_dgrad
        kp = (K - p + stride - 1) // stride
        d = pl - p
        u_min = (d + stride - 1) // stride if d > 0 else 0
        t0 = stride * u_min + p - pl
        n_u = (T - 1 - t0) // stride + 1 if t0 < T else 0
        total += mma_flops(B, n_u, Cin, kp * Cout, x3)
    return total


def time_us(fn, iters=50):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters * 1e3


def bench_shape(name, B, T, Cin, Cout, K, stride, pl, prec):
    capi.set_precision(prec)
    x3 = prec == "f32"
    g = torch.Generator(device="cuda").manual_seed(0)
    Tout = tout_of(T, K, stride, pl)
    x = torch.randn(B, T, Cin, W, device="cuda", generator=g)
    wt = torch.randn(Cout, Cin, K, device="cuda", generator=g) * 0.1
    bias = torch.randn(Cout, device="cuda", generator=g)
    dy = torch.randn(B, Tout, Cout, W, device="cuda", generator=g)
    y = torch.empty(B, Tout, Cout, W, device="cuda")
    dx = torch.empty(B, T, Cin, W, device="cuda")
    dwt, dbias = torch.zeros(Cout, Cin, K, device="cuda"), torch.zeros(Cout, device="cuda")
    ws = capi.conv_time_ws(B, Tout, Cin, Cout, K, x.device)
    s, lib, p = capi._stream, capi.lib, capi._ptr

    def fwd():
        capi._check(lib.w2l_conv_time_fwd(s(), B, T, Tout, W, Cin, Cout, K, stride, pl, p(x), p(wt), p(bias), None, p(y), 1, 0.2, 5,
                                          p(ws), ws.numel()))

    def dgrad():
        capi._check(lib.w2l_conv_time_dgrad(s(), B, T, Tout, W, Cin, Cout, K, stride, pl, p(dy), p(wt), None, p(dx), p(ws), ws.numel()))

    def wgrad():
        capi._check(lib.w2l_conv_time_wgrad(s(), B, T, Tout, W, Cin, Cout, K, stride, pl, p(x), p(dy), p(dwt), p(dbias), p(ws),
                                            ws.numel()))

    xb, yb = 4 * B * T * Cin * W, 4 * B * Tout * Cout * W
    rec = {"shape": name, "precision": prec, "B": B, "T": T, "Tout": Tout, "Cin": Cin, "Cout": Cout, "K": K, "stride": stride}
    for d, fn, nbytes, flops in (("fwd", fwd, xb + yb, mma_flops(B, Tout, Cout, K * Cin, x3)),
                                 ("dgrad", dgrad, yb + xb, dgrad_flops(B, T, Tout, Cin, Cout, K, stride, pl, x3)),
                                 ("wgrad", wgrad, xb + yb, mma_flops(B, Tout, Cout, (K * Cin + 7) // 8 * 8, x3))):
        us = time_us(fn)
        rec[d] = {"us": round(us, 1), "GBps": round(nbytes / us / 1e3, 1), "TFLOPs": round(flops / us / 1e6, 2)}
    return rec


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip() or torch.cuda.get_device_name(0)
    print(f"card: {card}", flush=True)
    out = {"card": card, "shapes": []}
    step = {}
    for prec in ("f32", "tf32"):
        tot = {"fwd": 0.0, "dgrad": 0.0, "wgrad": 0.0}
        for name, B, T, Cin, Cout, K, stride, pl, calls in SHAPES:
            rec = bench_shape(name, B, T, Cin, Cout, K, stride, pl, prec)
            out["shapes"].append(rec)
            print(json.dumps(rec), flush=True)
            if calls:
                for d, n in zip(("fwd", "dgrad", "wgrad"), calls):
                    tot[d] += n * rec[d]["us"]
        tot = {k: round(v, 1) for k, v in tot.items()}
        tot["total_us"] = round(sum(tot.values()), 1)
        step[prec] = tot
    capi.set_precision("tf32")
    out["seq2seq_step_conv_us"] = step
    print(json.dumps({"seq2seq_step_conv_us": step}), flush=True)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
