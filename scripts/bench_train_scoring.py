"""The cost of scoring training batches (Trainer.step(..., text=...), Train.cpp's meters.train): scored against unscored
training steps in one process, alternated in rounds so that clocks and neighbours affect both alike, on bench.py's
workloads:
  tds_ctc f32 / bf16   seq2seq_tds TDS + CTC, 10 000 word pieces (the argmax fused into the CTC prep pass)
  tds_asg              seq2seq_tds TDS + ASG, 28 letters + replabel 2 (FCC Viterbi on the scoring stream)
  conv_glu_asg         conv_glu 17-layer Conv1D+GLU + ASG, bf16
and Trainer.evaluate against step(train=False) (the eval loss alone) on the tds_ctc batch.  Inputs are bench.py's
(make_train_inputs); the text pipeline has the workload's class count.  Prints the card and its power limit, then one
JSON line per workload with the median step times over the rounds, their spread and the overhead."""
import argparse
import json
import os
import random
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from wav2letter_b200.text import TextPipeline  # noqa: E402
from wav2letter_b200.trainer import Trainer  # noqa: E402

LETTERS = "|\n'\n" + "\n".join("abcdefghijklmnopqrstuvwxyz") + "\n"


def text_for(cfg):
    if cfg["crit"] == "ctc":  # N - 1 word pieces; the pipeline appends the blank
        rng, alpha, pieces = random.Random(0), "abcdefghijklmnopqrstuvwxyz'", set()
        while len(pieces) < cfg["N"] - 1:
            pieces.add(("_" if rng.random() < 0.4 else "") + "".join(rng.choice(alpha) for _ in range(rng.randint(1, 6))))
        tp = TextPipeline("\n".join(sorted(pieces)) + "\n", "", "ctc", 0, "", True, "_")
    else:
        tp = TextPipeline(LETTERS, "", "asg", 2, "|", False, "|")
    assert tp.num_classes == cfg["N"], (tp.num_classes, cfg["N"])
    return tp


def timed(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(n):
        fn(i)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def run(name, precision, rounds, per_round, warmup):
    cfg = dict(bench.WORKLOADS[name])
    tp = text_for(cfg)
    tr = Trainer(cfg["arch"], cfg["F"], cfg["N"], cfg["crit"], cfg["scale_mode"], transdiag=cfg["transdiag"], lr=cfg["lr"], lrcrit=cfg["lrcrit"],
                 momentum=cfg["momentum"], maxgradnorm=cfg["maxgradnorm"], precision=precision)
    rng = np.random.default_rng(1234)
    sets = [tuple(torch.from_numpy(a).cuda() for a in bench.make_train_inputs(rng, cfg)) for _ in range(4)]
    B = cfg["B"]
    loss = torch.empty(B, device="cuda")

    def plain(i):
        f, y = sets[i % len(sets)]
        tr.step(f, y, True, float(B), loss)

    def scored(i):
        f, y = sets[i % len(sets)]
        tr.step(f, y, True, float(B), loss, text=tp)

    timed(plain, warmup)
    timed(scored, warmup)
    t_plain, t_scored = [], []
    for r in range(rounds):
        order = (plain, scored) if r % 2 == 0 else (scored, plain)
        for fn in order:
            (t_plain if fn is plain else t_scored).append(timed(fn, per_round))
    out = dict(workload=name, precision=precision, B=B, T=cfg["T"], N=cfg["N"], steps_each=rounds * per_round,
               plain_ms=float(np.median(t_plain)), scored_ms=float(np.median(t_scored)),
               plain_spread_ms=[float(min(t_plain)), float(max(t_plain))], scored_spread_ms=[float(min(t_scored)), float(max(t_scored))])
    out["overhead_pct"] = 100.0 * (out["scored_ms"] / out["plain_ms"] - 1.0)
    if name == "tds_ctc" and precision == "f32":  # validation: evaluate against the eval loss alone
        f, y = sets[0]
        t_eval, t_loss = [], []
        timed(lambda i: tr.evaluate(f, y, tp), warmup)
        for r in range(rounds):
            t_loss.append(timed(lambda i: tr.step(f, y, False, None, loss), per_round))
            t_eval.append(timed(lambda i: tr.evaluate(f, y, tp), per_round))
        out.update(eval_loss_ms=float(np.median(t_loss)), evaluate_ms=float(np.median(t_eval)))
    tr.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--per-round", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", default="", help="comma-separated workload[:precision] list (default: all)")
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi": smi.stdout.strip().splitlines()[:1]}), flush=True)
    runs = [("tds_ctc", "f32"), ("tds_ctc", "bf16"), ("tds_asg", "f32"), ("conv_glu_asg", "bf16")]
    if args.only:
        want = [w.split(":") for w in args.only.split(",")]
        runs = [r for r in runs if any(w[0] == r[0] and (len(w) == 1 or w[1] == r[1]) for w in want)]
    for name, precision in runs:
        print(json.dumps(run(name, precision, args.rounds, args.per_round, args.warmup)), flush=True)


if __name__ == "__main__":
    main()
