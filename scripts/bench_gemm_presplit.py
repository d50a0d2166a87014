"""F32X3 on a weight B, converted in every tile (kind f32x3), against the weight split once per call into tf32 hi / lo
planes (w2l_split_tf32) and read by TMA (kind f32x3_split_b), on the 8 forward and data-gradient shapes of the
seq2seq_tds step (those of bench_gemm_kinds.py; the weight gradients have no weight operand).  The two are timed
alternately, ROUNDS times, with inputs rotated over enough buffers to exceed the 50 MB L2; the split-B time includes
the split.  Prints one JSON record per shape (median µs), then the sums over one train step: each shape weighted by the
number of Linear layers that run it (2 per TDS block: 2, 3 and 6 blocks per stage, and the head)."""
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import wav2letter_b200 as w  # noqa: E402

SHAPES = [("stage1 fc", 9600, 800, 800, 4), ("stage2 fc", 4800, 1120, 1120, 6), ("stage3 fc", 2400, 1440, 1440, 12),
          ("head", 2400, 10000, 1440, 1)]
ROUNDS, ITERS = 5, 20


def main():
    dev = torch.cuda.get_device_properties(0)
    print(json.dumps({"device": dev.name, "sms": dev.multi_processor_count}), flush=True)
    recs, step = [], {"f32x3_us": 0.0, "split_b_us": 0.0, "split_us": 0.0}
    for name, rows, nout, nin, per_step in SHAPES:
        # forward Y[rows][nout] = X W^T (B = W K-major); dgrad dX[rows][nin] = dY W (B = W MN-major, split transposed)
        for op, (M, N, K, b_mn) in {"fwd": (rows, nout, nin, False), "dgrad": (rows, nin, nout, True)}.items():
            nbuf = max(2, int(200e6 // ((M * K + N * K + M * N) * 4)) + 1)
            As = [torch.randn(M, K, device="cuda") for _ in range(nbuf)]
            Ws = [torch.randn(nout, nin, device="cuda") for _ in range(nbuf)]  # the weight as the Linear stores it
            Cs = [torch.empty(M, N, device="cuda") for _ in range(nbuf)]

            def cur(i):
                w.capi.gemm(As[i], Ws[i], "f32x3", False, b_mn, out=Cs[i])

            def split(i):
                return w.capi.split_tf32(Ws[i], transpose=b_mn)

            def new(i):
                w.capi.gemm(As[i], split(i), "f32x3_split_b", out=Cs[i])

            ref = w.capi.gemm(As[0], Ws[0], "f32x3", False, b_mn)
            got = w.capi.gemm(As[0], split(0), "f32x3_split_b")
            identical = bool(torch.equal(ref, got))

            def timed(fn):
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                for i in range(ITERS):
                    fn(i % nbuf)
                t1.record()
                torch.cuda.synchronize()
                return t0.elapsed_time(t1) / ITERS * 1e3

            for fn in (cur, new, split):  # warm-up
                for i in range(3):
                    fn(i % nbuf)
            torch.cuda.synchronize()
            t = {"cur": [], "new": [], "split": []}
            for _ in range(ROUNDS):
                t["cur"].append(timed(cur))
                t["new"].append(timed(new))
                t["split"].append(timed(split))
            med = {k: statistics.median(v) for k, v in t.items()}
            rec = {"shape": name, "op": op, "M": M, "N": N, "K": K, "identical": identical, "f32x3_us": round(med["cur"], 2),
                   "split_b_us": round(med["new"], 2), "split_us": round(med["split"], 2),
                   "f32x3_range": [round(min(t["cur"]), 2), round(max(t["cur"]), 2)],
                   "split_b_range": [round(min(t["new"]), 2), round(max(t["new"]), 2)],
                   "f32x3_tflops": round(2.0 * M * N * K / med["cur"] / 1e6, 1),
                   "split_b_gemm_tflops": round(2.0 * M * N * K / (med["new"] - med["split"]) / 1e6, 1),
                   "saved": round(1.0 - med["new"] / med["cur"], 3)}
            recs.append(rec)
            print(json.dumps(rec), flush=True)
            step["f32x3_us"] += per_step * med["cur"]
            step["split_b_us"] += per_step * med["new"]
            step["split_us"] += per_step * med["split"]
            del As, Ws, Cs
            torch.cuda.empty_cache()
    step = {k: round(v, 1) for k, v in step.items()}
    step["saved"] = round(1.0 - step["split_b_us"] / step["f32x3_us"], 3)
    shapes_sum = {"f32x3_us": round(sum(r["f32x3_us"] for r in recs), 1), "split_b_us": round(sum(r["split_b_us"] for r in recs), 1)}
    shapes_sum["saved"] = round(1.0 - shapes_sum["split_b_us"] / shapes_sum["f32x3_us"], 3)
    print(json.dumps({"sum_over_8_shapes": shapes_sum, "per_step": step}), flush=True)


if __name__ == "__main__":
    main()
