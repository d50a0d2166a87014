"""Step time and GEMM rate of the tds_ctc and streaming_tds_ctc training steps in bf16 and in fp16 GEMM operands.

The method is bench.py's (its workloads, inputs, Timed.run: warm-up steps, then K steps between synchronisations timed
with CUDA events, the wgmma GEMM launches of the first three timed steps timed by the profile event list).  The two
precisions run alternately, `--reps` times each, in one process; the medians are reported with the card's name, power
limit and the SM clocks sampled during the timed steps.  GEMM TFLOP/s = bench.arch_gemm_flops (2MNK of every dense
contraction, forward + both gradients) over the summed GEMM kernel time of a step.

    python scripts/bench_fp16.py --steps 20 --warmup 3 [--reps 3] [--out result.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

PRECISIONS = ("bf16", "fp16")


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return {"error": str(e)}
    name, power, clock = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def measure(workload, steps, warmup, reps):
    import torch

    from wav2letter_b200 import capi
    from wav2letter_b200.trainer import Trainer

    cfg = dict(bench.WORKLOADS[workload])
    B, T = cfg["B"], cfg["T"]
    tm = bench.Timed(1, 0)
    trainers = {p: Trainer(cfg["arch"], cfg["F"], cfg["N"], cfg["crit"], cfg["scale_mode"], transdiag=cfg["transdiag"], lr=cfg["lr"],
                           lrcrit=cfg["lrcrit"], momentum=cfg["momentum"], maxgradnorm=cfg["maxgradnorm"], precision=p)
                for p in PRECISIONS}
    rng = np.random.default_rng(1234)
    inputs = []
    for _ in range(cfg["n_input_sets"]):
        f, y = bench.make_train_inputs(rng, cfg)
        inputs.append((torch.from_numpy(f).cuda(), torch.from_numpy(y).cuda()))
    loss = torch.empty(B, dtype=torch.float32, device="cuda")
    flops, _ = bench.arch_gemm_flops(cfg["arch"], B, T, cfg["F"], cfg["N"])
    prof_steps = min(steps, 3)
    runs = {p: [] for p in PRECISIONS}
    clocks = {p: [] for p in PRECISIONS}
    for _ in range(reps):
        for p in PRECISIONS:
            tr = trainers[p]

            def step(i):
                f, y = inputs[i % len(inputs)]
                tr.step(f, y, True, float(B), loss)

            prof = capi.ProfileList(1, 400 * prof_steps)
            ms, kern, _, clk = tm.run(step, steps, warmup, sample_clocks=True, profile=prof, profile_steps=prof_steps)
            runs[p].append((ms / steps, sum(kern) / prof_steps))
            clocks[p].append(clk)
    out = {}
    for p in PRECISIONS:
        step_ms = statistics.median(r[0] for r in runs[p])
        gemm_ms = statistics.median(r[1] for r in runs[p])
        out[p] = {"ms_per_step": step_ms, "frames_per_sec": B * T / (step_ms * 1e-3), "gemm_ms_per_step": gemm_ms,
                  "gemm_tflops": flops / (gemm_ms * 1e-3) / 1e12, "ms_per_step_runs": [round(r[0], 3) for r in runs[p]],
                  "skipped_steps": trainers[p].skipped_steps(), "clocks": clocks[p]}
        trainers[p].close()
    out["fp16_over_bf16_step_time"] = out["fp16"]["ms_per_step"] / out["bf16"]["ms_per_step"]
    out["workload"] = bench.train_workload_text(cfg)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workloads", nargs="+", default=["tds_ctc", "streaming_tds_ctc"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_fp16: needs a CUDA device")
    res = {"card": card(), "steps": args.steps, "warmup": args.warmup, "reps": args.reps}
    for w in args.workloads:
        res[w] = measure(w, args.steps, args.warmup, args.reps)
    line = json.dumps(res)
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
