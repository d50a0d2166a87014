"""Serial against concurrent timing of each backward GEMM pair of the seq2seq_tds train step in f32x3: the data gradient
dX = dY W and the weight gradient dW = dY^T X of one fully-connected layer (and of the 10 000-class head), first one
after the other on one stream, then on two streams (the weight gradient on a low-priority stream, as the trainer runs
it).  Inputs rotate over enough buffers to exceed the 50 MB L2.  Prints one JSON record per pair, then the list."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import wav2letter_b200 as w  # noqa: E402

# (name, rows = frames of the batch, nout, nin) of the Linear layers; B = 16 x T = 1200 frames, strides 2, 2, 2
SHAPES = [("stage1 fc", 9600, 800, 800), ("stage2 fc", 4800, 1120, 1120), ("stage3 fc", 2400, 1440, 1440), ("head", 2400, 10000, 1440)]


def time_pair(rows, nout, nin, kind="f32x3", iters=20):
    nbuf = max(2, int(200e6 // (4 * (2 * rows * nout + 2 * rows * nin + nout * nin))) + 1)
    dY = [torch.randn(rows, nout, device="cuda") for _ in range(nbuf)]
    X = [torch.randn(rows, nin, device="cuda") for _ in range(nbuf)]
    W = [torch.randn(nout, nin, device="cuda") for _ in range(nbuf)]
    dX = [torch.empty(rows, nin, device="cuda") for _ in range(nbuf)]
    dW = [torch.empty(nout, nin, device="cuda") for _ in range(nbuf)]
    side = torch.cuda.Stream(priority=0)  # 0 is the lowest stream priority
    main = torch.cuda.current_stream()

    def dgrad(i):
        w.capi.gemm(dY[i], W[i], kind, False, True, out=dX[i])

    def wgrad(i):
        w.capi.gemm(dY[i], X[i], kind, True, True, out=dW[i])

    def run(concurrent):
        for i in range(iters):
            k = i % nbuf
            if concurrent:
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    wgrad(k)
            else:
                wgrad(k)
            dgrad(k)
        if concurrent:
            main.wait_stream(side)

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        fn()
        t1.record()
        torch.cuda.synchronize()
        return t0.elapsed_time(t1) / iters * 1e3  # us per pair

    def alone(fn):
        return timed(lambda: [fn(i % nbuf) for i in range(iters)])

    return alone(dgrad), alone(wgrad), timed(lambda: run(False)), timed(lambda: run(True))


def main():
    out = []
    for name, rows, nout, nin in SHAPES:
        d_us, w_us, serial_us, conc_us = time_pair(rows, nout, nin)
        rec = {"shape": name, "dgrad": [rows, nin, nout], "wgrad": [nout, nin, rows], "dgrad_us": round(d_us, 1), "wgrad_us": round(w_us, 1),
               "serial_us": round(serial_us, 1), "concurrent_us": round(conc_us, 1), "saved_us": round(serial_us - conc_us, 1),
               "saved_frac": round(1 - conc_us / serial_us, 3)}
        out.append(rec)
        print(json.dumps(rec), flush=True)
    json.dump(out, sys.stdout, indent=1)


if __name__ == "__main__":
    main()
