"""Scoring a dev set: per-utterance host scoring (prediction2ltr / target2ltr / ltr2wrd / EditDistanceMeter after a copy
to the host, today's Python route) against TextPipeline.edit_counts on the GPU, over the same paths.

2 700 utterances with LibriSpeech-dev-like durations (1.5-33 s, mean ~7 s), in batches of --batch.  Paths are
synthetic and early-training-shaped: long and wrong.
  ctc      10 000 word pieces, usewordpiece, 8x time stride (one path entry per 80 ms), every token a random piece
           or blank
  asg      28 letters + replabel 2 + surround "|", one entry per 10 ms frame, random letters in runs
  seq2seq  10 000 word pieces, decode rows of up to 200 tokens with eos
Prints one JSON line per setting: both times, the counts' equality and the kernels' time per million DP cells
(letter cells plus word cells).  The acoustic model's forward is not included in either time.

--trainer runs the whole validation pass instead, on the seq2seq_tds TDS acoustic model (80 filterbanks, 8x stride,
untrained: its paths are long and wrong) over the same 2 700 durations, batches of --batch sorted by length:
  ctc  10 000 word pieces;  asg  28 letters + replabel 2 + surround "|"
Method A is what a Python caller does today: step(train=False) for the loss, viterbi_path, a copy to the host and
per-utterance host scoring.  Method B is Trainer.evaluate.  Also reported: viterbi_path alone (forward and path)."""
import argparse
import json
import os
import random
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from wav2letter_b200.text import EditDistanceMeter, TextPipeline  # noqa: E402


def wordpieces(n, rng):
    alpha = "abcdefghijklmnopqrstuvwxyz'"
    out, seen = [], set()
    while len(out) < n:
        w = ("_" if rng.random() < 0.4 else "") + "".join(rng.choice(alpha) for _ in range(rng.randint(1, 6)))
        if w not in seen:
            seen.add(w)
            out.append(w)
    return out


def durations(rng, n):
    return [min(33.0, max(1.5, rng.lognormvariate(1.75, 0.6))) for _ in range(n)]


def setting(name, rng, n_utt):
    if name == "asg":
        tokens = ["|", "'"] + list("abcdefghijklmnopqrstuvwxyz")
        tp = TextPipeline("\n".join(tokens) + "\n", "", "asg", 2, "|", False, "|")
    else:
        tokens = wordpieces(10000, rng)
        tp = TextPipeline("\n".join(tokens) + "\n", "", "ctc" if name == "ctc" else "seq2seq", 0, "", True, "_")
    N = tp.num_classes
    paths, targets = [], []
    for d in durations(rng, n_utt):
        words = max(1, int(d * 2.7))
        if name == "asg":
            tgt = tp.encode(" ".join("".join(rng.choice("abcdefghij") for _ in range(rng.randint(2, 8))) for _ in range(words)))
            T = int(d * 100)
            p = []
            while len(p) < T:
                p += [rng.randrange(N)] * rng.randint(1, 6)
            path = p[:T]
        else:
            tgt = np.array([rng.randrange(len(tokens)) for _ in range(int(words * 1.5))], np.int32)
            if name == "ctc":
                T = int(d * 100 / 8)
                path = [rng.randrange(N) if rng.random() < 0.6 else N - 1 for _ in range(T)]
            else:
                tgt = np.append(tgt, N - 2)
                n = min(200, int(len(tgt) * rng.uniform(0.5, 2.0)) + 1)
                path = [rng.randrange(len(tokens)) for _ in range(n - 1)] + [N - 2]
        paths.append(path)
        targets.append(list(tgt))
    return tp, paths, targets


def pad(rows, fill):
    a = np.full((len(rows), max(1, max(len(r) for r in rows))), fill, np.int32)
    for b, r in enumerate(rows):
        a[b, :len(r)] = r
    return a


def host_score(tp, paths, targets):
    out = []
    for p, q in zip(paths.cpu().numpy(), targets.cpu().numpy()):
        hl, rl = tp.prediction2ltr(p), tp.target2ltr(q)
        ml, mw = EditDistanceMeter(), EditDistanceMeter()
        ml.add(hl, rl)
        mw.add(tp.ltr2wrd(hl), tp.ltr2wrd(rl))
        out.append(list(ml.raw()) + list(mw.raw()))
    return out


def trainer_mode(args, props):
    from wav2letter_b200 import archs
    from wav2letter_b200.trainer import Trainer

    F = 80
    for name in args.settings.split(","):
        if name not in ("ctc", "asg"):
            continue
        rng = random.Random(7)
        if name == "asg":
            tp = TextPipeline("\n".join(["|", "'"] + list("abcdefghijklmnopqrstuvwxyz")) + "\n", "", "asg", 2, "|", False, "|")
        else:
            tp = TextPipeline("\n".join(wordpieces(10000, rng)) + "\n", "", "ctc", 0, "", True, "_")
        N = tp.num_classes
        tr = Trainer(archs.seq2seq_tds(ctc_head=True), F, N, name, "none", transdiag=0.0, lr=0.0)
        durs = sorted(durations(rng, args.utterances))
        gen = torch.Generator(device="cuda").manual_seed(0)
        batches = []
        for i in range(0, len(durs), args.batch):
            ds = durs[i:i + args.batch]
            T = int(max(ds) * 100)
            feat = torch.randn((len(ds), 1, F, T), generator=gen, device="cuda")
            rows = [list(rng.randrange(N - (1 if name == "ctc" else 2)) for _ in range(max(1, int(d * 2.7 * 1.5)))) for d in ds]
            if name == "asg":
                rows = [list(tp.encode(" ".join("".join(rng.choice("abcdefghij") for _ in range(rng.randint(2, 5))) for _ in range(max(1, int(d * 2.0)))))) for d in ds]
            batches.append((feat, torch.from_numpy(pad(rows, -1)).cuda()))
        for feat, tgt in batches[-2:]:  # warm up the longest shapes
            tr.evaluate(feat, tgt, tp)
            tr.viterbi_path(feat)
        torch.cuda.synchronize()
        times, results = {}, {}
        for method in ("A", "B", "path", "A", "B", "path"):  # alternated, the second round reported
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = []
            for feat, tgt in batches:
                if method == "A":
                    tr.step(feat, tgt, train=False)
                    res += host_score(tp, tr.viterbi_path(feat), tgt)
                elif method == "B":
                    res.append(tr.evaluate(feat, tgt, tp)[1])
                else:
                    res.append(tr.viterbi_path(feat))
            if method == "B":
                res = torch.cat(res).cpu().numpy().tolist()
            torch.cuda.synchronize()
            times[method] = time.perf_counter() - t0
            results[method] = res
        print(json.dumps({"mode": "trainer", "setting": name, "utterances": len(durs), "batch": args.batch,
                          "A_step_eval_path_host_score_s": round(times["A"], 4), "B_evaluate_s": round(times["B"], 4),
                          "viterbi_path_only_s": round(times["path"], 4), "equal": results["A"] == results["B"], "gpu": props.name}), flush=True)
        tr.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utterances", type=int, default=2700)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--settings", default="ctc,asg,seq2seq")
    ap.add_argument("--trainer", action="store_true", help="the whole validation pass: forward, loss, path and scoring")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_eval measures on the GPU"
    props = torch.cuda.get_device_properties(0)
    if args.trainer:
        trainer_mode(args, props)
        return
    for name in args.settings.split(","):
        rng = random.Random(7)
        tp, paths, targets = setting(name, rng, args.utterances)
        fill = tp.pad_index
        batches = [(torch.from_numpy(pad(paths[i:i + args.batch], fill)).cuda(), torch.from_numpy(pad(targets[i:i + args.batch], fill)).cuda())
                   for i in range(0, len(paths), args.batch)]
        tp.edit_counts(*batches[0])  # tables and first launch
        torch.cuda.synchronize()
        # method A: copy each batch's paths to the host and score utterance by utterance
        t0 = time.perf_counter()
        host, cells = [], 0
        for P, Tg in batches:
            Pc, Tc = P.cpu().numpy(), Tg.cpu().numpy()
            for p, q in zip(Pc, Tc):
                hl, rl = tp.prediction2ltr(p), tp.target2ltr(q)
                hw, rw = tp.ltr2wrd(hl), tp.ltr2wrd(rl)
                ml, mw = EditDistanceMeter(), EditDistanceMeter()
                ml.add(hl, rl)
                mw.add(hw, rw)
                host.append(list(ml.raw()) + list(mw.raw()))
                cells += len(hl) * len(rl) + len(hw) * len(rw)
        t_host = time.perf_counter() - t0
        # method B: the device scoring of every batch, one read-back at the end
        for _ in range(2):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            dev = [tp.edit_counts(P, Tg) for P, Tg in batches]
            stop.record()
            got = torch.cat(dev).cpu().numpy()
            t_dev = time.perf_counter() - t0
        ms = start.elapsed_time(stop)
        print(json.dumps({"setting": name, "utterances": len(paths), "batch": args.batch, "host_s": round(t_host, 4),
                          "device_s": round(t_dev, 4), "device_events_ms": round(ms, 3), "equal": bool(np.array_equal(got, np.array(host))),
                          "dp_cells_M": round(cells / 1e6, 2), "ms_per_M_cells": round(ms / max(cells / 1e6, 1e-9), 4),
                          "gpu": props.name}), flush=True)


if __name__ == "__main__":
    main()
