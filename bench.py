#!/usr/bin/env python
"""bench.py — measurement contract of the repo (task statement, "Measurement").

    python bench.py --gpus N --steps K --warmup W [--impl reference] [--workload W] [--precision P] [--dump-outputs DIR]

Workloads (one full TRAIN STEP per step unless noted: network forward, criterion, backward, NCCL gradient all-reduce
for N > 1, division by the global batch, NaN/Inf guard, clipGradNorm, SGD; data parallel by utterance = weak scaling,
the gradient all-reduce is the only collective — SURVEY.md §8e):
  tds_ctc (default)  BASELINE.json configs[1]: seq2seq_tds LibriSpeech TDS acoustic model + CTC, "fp32": B=16 utterances
                     x T=1200 filterbank frames (80 bins) per GPU, 10 000 word-piece classes, targets <= 60 tokens
                     (recipes/seq2seq_tds/librispeech/train.cfg: batchsize 16, lr 0.05, maxgradnorm 15).
  conv_glu_asg       configs[2]: conv_glu LibriSpeech 17-layer Conv1D+GLU model (209 M parameters) + ASG, "bf16 convs /
                     fp32 loss": B=8 x T=1000 x 40 filterbanks per GPU, 30 letters.
  streaming_tds_ctc  configs[3]: streaming_convnets TDS (am_500ms_future_context.arch) + CTC, 10 s chunks, "bf16":
                     B=8 x T=1000 x 80 per GPU, 10 000 word pieces (train_am_500ms_future_context.cfg: batchsize 8).
  asg                configs[4] point: fused ASG forward+backward at T=1500, N=30, B=64 per GPU (no train step).
  asg_sweep          configs[4]: T in {100,500,1500,4000} x B in {1,16,64,256} per GPU, oracle parity on every point.
--precision: f32 (fp32-accurate: error-compensated 3xTF32 wgmma GEMMs and time convolutions), tf32, bf16 (bf16 GEMM operands,
fp32 accumulation / LayerNorm / criterion / optimizer); default = the precision the workload's BASELINE config states.

One JSON line on rank 0.  `value` = frames/s with the batch resident in HBM; `e2e` = the same step through the C ABI
with HOST (pinned) batches, H2D of features/targets and D2H of the losses inside the timed region; `roofline` = the
dominant kernel (train steps: gemm_wgmma_kernel, achieved algorithmic TFLOP/s over all GEMM launches of the timed
steps; asg: asg_chains_kernel GB/s) timed live with CUDA events through w2l_set_profile_event_list against
MEASURED_PEAKS.json; `cpu_baseline` = the CPU port (oracle/) timed on this box's host cores.  The default workload
also reports the other precisions of the same step, the TDS+ASG step BASELINE.json's metric names, and the ASG point.
`--impl reference` times the CPU implementation as the reference arm (the reference's own ArrayFire-CPU backend cannot
be built here: DESIGN.md §2): same config (B, T, arch) as the GPU arm, all host threads it can use.
`--dump-outputs DIR` writes, after the timed steps, what the timed path computed in its last step as DIR/<name>.npy
(float32; arrays above 4 M elements as a fixed, seeded sample of 4 M, named <name>_sample.npy): the per-utterance losses
and the parameters after the update for the train steps; loss, d_emis and d_trans for the ASG workloads (asg_sweep: the
T=1500, B=64 point).  The inputs are seeded, so two builds can be compared output for output.
"""
from __future__ import annotations

import argparse
import importlib.util
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def load_archs():
    """wav2letter_b200/archs.py by path: the reference arm must not map the CUDA library into its process"""
    spec = importlib.util.spec_from_file_location("w2l_archs", os.path.join(ROOT, "wav2letter_b200", "archs.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


ARCHS = load_archs()
ASG_CFG = dict(T=1500, N=30, B=64, L=250, scale_mode="target_sz_sqrt", n_input_sets=16)
WORKLOADS = {
    "tds_ctc": dict(arch=ARCHS.seq2seq_tds(True), crit="ctc", scale_mode="none", transdiag=0.0, B=16, T=1200, F=80, N=10000, L=60,
                    lr=0.05, lrcrit=0.0, momentum=0.0, maxgradnorm=15.0, precision="f32", n_input_sets=8,
                    desc="seq2seq_tds LibriSpeech TDS acoustic model + CTC (BASELINE.json configs[1]; "
                         "recipes/seq2seq_tds/librispeech/{network.arch,train.cfg})"),
    "tds_asg": dict(arch=ARCHS.seq2seq_tds(True), crit="asg", scale_mode="target_sz_sqrt", transdiag=4.0, B=16, T=1200, F=80, N=30, L=100,
                    lr=0.05, lrcrit=0.001, momentum=0.0, maxgradnorm=15.0, precision="f32", n_input_sets=8,
                    desc="seq2seq_tds TDS acoustic model + ASG over 30 letters (the step BASELINE.json's metric words: TDS+ASG)"),
    "conv_glu_asg": dict(arch=ARCHS.conv_glu_librispeech(), crit="asg", scale_mode="target_sz_sqrt", transdiag=4.0, B=8, T=1000, F=40, N=30,
                         L=160, lr=0.1, lrcrit=0.001, momentum=0.0, maxgradnorm=0.2, precision="bf16", n_input_sets=4,
                         desc="conv_glu LibriSpeech 17-layer Conv1D+GLU acoustic model (WeightNorm) + ASG (BASELINE.json configs[2]; "
                              "recipes/conv_glu/librispeech/{network.arch,train.cfg})"),
    "streaming_tds_ctc": dict(arch=ARCHS.streaming_tds(), crit="ctc", scale_mode="none", transdiag=0.0, B=8, T=1000, F=80, N=10000, L=60,
                              lr=0.4, lrcrit=0.0, momentum=0.0, maxgradnorm=0.5, precision="bf16", n_input_sets=8,
                              desc="streaming_convnets TDS (am_500ms_future_context.arch, SpecAugment on) + CTC, 10 s chunks "
                                   "(BASELINE.json configs[3]; recipes/streaming_convnets/librispeech/)"),
}
DTYPE_NOTE = {
    "f32": "f32 storage and fp32-ACCURATE contractions: the wgmma GEMMs split every staged operand tile into tf32 hi + lo parts and "
           "accumulate Al*Bh + Ah*Bl + Ah*Bh in fp32 registers (products good to ~2^-21); time convolutions on the mma.sync kernels with the same 3xTF32 split in registers; "
           "criterion / LayerNorm / optimizer in f32/f64",
    "tf32": "f32 storage; dense contractions multiply TF32 operands on the tensor cores with f32 accumulation (cuDNN / cuBLAS default for "
            "fp32 tensors); criterion, LayerNorm, optimizer in f32/f64",
    "bf16": "bf16 GEMM operands (activations and weights cast by their producers), fp32 accumulation in registers; fp32 master weights, "
            "LayerNorm, criterion (fp32 loss) and optimizer: the reference's AMP mode (Train.cpp:211-219) with bf16",
}


def asg_algorithmic_bytes(B, T, N, L):
    """SURVEY.md §8(d): read emis + write d_emis + trans/d_trans + targets + losses."""
    return 8 * B * T * N + 8 * N * N + 4 * B * L + 4 * B


def arch_gemm_flops(arch_text, B, T, n_feat, n_label):
    """2*M*N*K summed over every dense contraction that runs on the wgmma GEMM (TDS fully-connected layers, Linear layers,
    the WN Conv1D layers of the conv_glu archs as im2col GEMMs), x3 (forward, data gradient, weight gradient).
    Returns (flops per step, output frames)."""
    total, t, pend = 0, T, None
    for line in arch_text.splitlines():
        p = line.split("#")[0].replace("NFEAT", str(n_feat)).replace("NLABEL", str(n_label)).split()
        if not p:
            continue
        if p[0] == "PD":
            pend = (int(p[2]), int(p[3]))
        elif p[0] == "C2":
            k, s = int(p[3]), int(p[5])
            px = int(p[7]) if len(p) > 7 else 0
            if pend is not None:
                pl, pr = pend
                pend = None
            elif px == -1:
                rem = t % s
                pl = pr = max(((k - 1) - (s if rem == 0 else rem) + 1 + 1) // 2, 0)
            else:
                pl = pr = px
            t = (t + pl + pr - k) // s + 1
        elif p[0] == "TDS":
            d = int(p[1]) * int(p[3])
            inner = int(p[5]) if len(p) > 5 and int(p[5]) > 0 else d
            total += 2 * (2 * B * t * d * inner)
        elif p[0] == "L":
            total += 2 * B * t * int(p[1]) * int(p[2])
        elif p[0] == "WN" and p[2] in ("C", "C1"):
            cin, cout, kw, pad = int(p[3]), int(p[4]), int(p[5]), (int(p[7]) if len(p) > 7 else 0)
            t = t + 2 * ((kw // 2) if pad == -1 else pad) - kw + 1
            total += 2 * B * t * cout * cin * kw
        elif p[0] == "WN" and p[2] == "L":
            total += 2 * B * t * int(p[3]) * int(p[4])
    return 3 * total, t


def make_asg_inputs(rng, B, T, N, L):
    e = (rng.standard_normal((B, T, N), dtype=np.float32) * 3).astype(np.float32)
    tr = (4 * np.eye(N) + rng.normal(0, 0.1, (N, N))).astype(np.float32)
    y = rng.integers(0, N, (B, L)).astype(np.int32)
    lens = rng.integers(max(1, T // 8), max(2, T // 5 + 1), B)
    lens = np.minimum(lens, L)
    for b in range(B):
        y[b, lens[b]:] = -1
    return e, tr, y


def make_train_inputs(rng, cfg, B=None):
    """features [B,1,F,T] (== ArrayFire [T,F,1,B]): x ~ N(0,1) (post-LocalNorm statistics); int targets, -1 padded."""
    B = B or cfg["B"]
    feat = rng.standard_normal((B, 1, cfg["F"], cfg["T"]), dtype=np.float32)
    hi = cfg["N"] - 1 if cfg["crit"] == "ctc" else cfg["N"]
    tgt = rng.integers(0, hi, (B, cfg["L"])).astype(np.int32)
    lens = rng.integers(cfg["L"] // 2, cfg["L"] + 1, B)
    for b in range(B):
        tgt[b, lens[b]:] = -1
    return feat, tgt


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
         "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int):
        self.idx = gpu_index
        self.rows = []
        self.proc = None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-i", str(self.idx), "-lms", "100"], stdout=subprocess.PIPE, text=True)
            threading.Thread(target=self._read, daemon=True).start()
            time.sleep(0.25)
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        sm = [float(r[1]) for r in self.rows if len(r) >= 9 and r[1].replace(".", "").isdigit()]
        mx = [float(r[2]) for r in self.rows if len(r) >= 9 and r[2].replace(".", "").isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = sorted({n for r in self.rows if len(r) >= 9 for n, v in zip(names, r[5:9]) if v.lower().startswith("active")})
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": reasons, "samples": len(sm)}


def measured_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d, "measured (MEASURED_PEAKS.json)"
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0}, "fallback: NVIDIA H100 SXM data sheet (700 W), not measured"


# ---------------------------------------------------------------------------------------------------------
# reference arm / CPU baselines (oracle/ is only ever used here, in tests/ and in smoke())
# ---------------------------------------------------------------------------------------------------------
def cpu_asg(sample_B, cfg, reps=3):
    os.environ["W2L_ORACLE_NATIVE"] = "1"  # -march=native build for THIS host (BASELINE.md §4)
    import oracle

    oracle.set_num_threads(os.cpu_count() or 1)
    rng = np.random.default_rng(99)
    e, tr, y = make_asg_inputs(rng, sample_B, cfg["T"], cfg["N"], cfg["L"])
    oracle.asg(e[:2], y[:2], tr, cfg["scale_mode"])
    best = 1e30
    for _ in range(reps):
        t0 = time.perf_counter()
        oracle.asg(e, y, tr, cfg["scale_mode"])
        best = min(best, time.perf_counter() - t0)
    return sample_B * cfg["T"] / best, best, oracle.num_threads()


class CpuArm:
    """torch-CPU (oneDNN) fp32 acoustic model + C-oracle criterion train step of the SAME arch / batch as the GPU arm."""

    def __init__(self, cfg):
        os.environ["W2L_ORACLE_NATIVE"] = "1"
        import oracle
        import torch
        from oracle.cpu_train import CpuTrainer

        self.cfg, self.torch, self.oracle = cfg, torch, oracle
        self.make = lambda threads: CpuTrainer(cfg["arch"], cfg["F"], cfg["N"], cfg["crit"], cfg["scale_mode"], cfg["transdiag"], cfg["lr"],
                                               cfg["lrcrit"], cfg["momentum"], cfg["maxgradnorm"], threads=threads)
        self.ncpu = os.cpu_count() or 1

    def pick_threads(self, feat, tgt):
        """all host threads — unless fewer are faster (oneDNN + OpenMP thrash on many-core hosts): one timed step of a
        B=2 sample per candidate, smallest first, stopping as soon as more threads stop helping; the sweep is reported"""
        cands = sorted({c for c in (16, 32, 64, self.ncpu) if c <= self.ncpu} | {min(self.ncpu, 16)})
        sweep, best = {}, None
        for c in cands:
            self.oracle.set_num_threads(c)
            tr = self.make(c)
            tr.step(feat[:2], tgt[:2])
            t0 = time.perf_counter()
            tr.step(feat[:2], tgt[:2])
            sweep[c] = round(time.perf_counter() - t0, 3)
            if best is None or sweep[c] < sweep[best]:
                best = c
            elif sweep[c] > 1.5 * sweep[best]:  # clearly past the optimum
                break
        return best, sweep

    def run(self, steps, warmup, budget_s=150.0):
        cfg = self.cfg
        rng = np.random.default_rng(4321)
        feat, tgt = make_train_inputs(rng, cfg)
        threads, sweep = self.pick_threads(feat, tgt)
        self.oracle.set_num_threads(threads)
        tr = self.make(threads)
        # per-step sample: the GPU arm's own batch unless the whole run would exceed the budget; then the largest power-of-two
        # fraction of it that fits (frames/s is per frame, the CPU port's cost is linear in B)
        t0 = time.perf_counter()
        tr.step(feat[:2], tgt[:2])
        est = (time.perf_counter() - t0) * cfg["B"] / 2
        B = cfg["B"]
        while B > 2 and est * B / cfg["B"] * (steps + warmup) > budget_s:
            B //= 2
        for _ in range(warmup):
            tr.step(feat[:B], tgt[:B])
        t0 = time.perf_counter()
        for _ in range(steps):
            tr.step(feat[:B], tgt[:B])
        dt = (time.perf_counter() - t0) / steps
        return dict(fps=B * cfg["T"] / dt, s_per_step=dt, threads=threads, sweep=sweep, B=B, same_batch=(B == cfg["B"]))


def run_reference(args, rank, world):
    """Reference arm: the CPU implementation of the path on this box's host cores (rank 0 only)."""
    if rank != 0:
        return
    wl = args.workload
    if wl in ("asg", "asg_sweep"):
        os.environ["W2L_ORACLE_NATIVE"] = "1"
        import oracle

        cfg = dict(ASG_CFG)
        oracle.set_num_threads(os.cpu_count() or 1)
        rng = np.random.default_rng(1234)
        e, tr, y = make_asg_inputs(rng, cfg["B"], cfg["T"], cfg["N"], cfg["L"])
        for _ in range(max(1, args.warmup)):
            oracle.asg(e, y, tr, cfg["scale_mode"])
        t0 = time.perf_counter()
        for _ in range(args.steps):
            oracle.asg(e, y, tr, cfg["scale_mode"])
        dt = (time.perf_counter() - t0) / args.steps
        fps, threads = cfg["B"] * cfg["T"] / dt, oracle.num_threads()
        workload = "ASG criterion fwd+bwd, T=1500 N=30 B=64 L<=250 per GPU (BASELINE.json configs[4] point)"
        sample = f"{args.steps} full batches of B=64,T=1500,N=30"
        extra = {}
    else:
        cfg = WORKLOADS[wl]
        r = CpuArm(cfg).run(args.steps, min(args.warmup, 1))
        fps, dt, threads = r["fps"], r["s_per_step"], r["threads"]
        workload = train_workload_text(cfg)
        sample = (f"{args.steps} train steps of B={r['B']} x T={cfg['T']}"
                  + ("" if r["same_batch"] else f" (bounded sample of the GPU arm's B={cfg['B']}: the run must end within minutes)"))
        extra = {"thread_sweep_s_per_step_B2": r["sweep"], "same_batch_as_gpu_arm": r["same_batch"]}
    line = {
        "impl": "reference", "metric": "frames_per_sec", "value": fps, "unit": "frames/s", "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 * dt, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": workload,
                   "note": "the reference's ArrayFire-CPU backend is unbuildable here (SURVEY.md §0); this is the CPU port: "
                           "torch-CPU/oneDNN fp32 for the acoustic-model operators + the C oracle (flashlight-0.3 "
                           "lib/sequence/criterion/cpu restated, -O3 -march=native -fopenmp) for the criterion", **extra},
        "cpu_baseline": {"value": fps, "unit": "frames/s", "cores": threads, "kind": "port", "sample": sample},
        "e2e": {"value": fps, "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    print(json.dumps(line), flush=True)


def train_workload_text(cfg):
    return (f"{cfg['desc']}, full train step (fwd, {cfg['crit'].upper()}, bwd, all-reduce, clip, SGD), B={cfg['B']} x T={cfg['T']} frames x "
            f"{cfg['F']} filterbanks per GPU, {cfg['N']} classes, targets <= {cfg['L']}")


# ---------------------------------------------------------------------------------------------------------
# GPU arms
# ---------------------------------------------------------------------------------------------------------
class Timed:
    def __init__(self, world, local_rank):
        import torch
        import torch.distributed as dist

        self.torch, self.dist, self.world, self.dev = torch, dist, world, torch.device("cuda", local_rank)
        self.local_rank = local_rank

    def barrier(self):
        if self.world > 1:
            self.dist.barrier()
        self.torch.cuda.synchronize()

    def run(self, fn, steps, warmup, sample_clocks=False, profile=None, profile_steps=3):
        """W warm-up steps, then exactly K steps between barrier+synchronize on both sides; device time, max over ranks."""
        import wav2letter_b200 as w

        torch = self.torch
        for i in range(warmup):
            fn(i)
        self.barrier()
        sampler = ClockSampler(self.local_rank) if sample_clocks else None
        if sampler:
            sampler.start()
        w.reset_launch_count()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        used = 0
        t0.record()
        for i in range(steps):
            if profile is not None and i == 0:
                profile.arm()
            fn(warmup + i)
            if profile is not None and i == profile_steps - 1:
                used = profile.disarm()
        if profile is not None and steps < profile_steps:
            used = profile.disarm()
        t1.record()
        self.barrier()
        launches = w.launch_count()
        clocks = sampler.stop() if sampler else None
        ms = t0.elapsed_time(t1)
        if self.world > 1:
            tms = torch.tensor([ms], device=self.dev)
            self.dist.all_reduce(tms, op=self.dist.ReduceOp.MAX)
            ms = float(tms.item())
        kern = profile.times_ms(used) if profile is not None else []
        return ms, kern, launches, clocks


DUMP_MAX_ELEMENTS = 4 << 20


def dump_outputs(out_dir, arrays):
    """DIR/<name>.npy in float32; an array above DUMP_MAX_ELEMENTS is written as a fixed, seeded sample of that many
    elements (sorted flat indices, DIR/<name>_sample.npy) so the files stay small but comparable run to run"""
    os.makedirs(out_dir, exist_ok=True)
    for name, t in arrays.items():
        a = t.detach().float().cpu().numpy().reshape(-1) if hasattr(t, "detach") else np.asarray(t, dtype=np.float32).reshape(-1)
        if a.size > DUMP_MAX_ELEMENTS:
            idx = np.sort(np.random.default_rng(0).choice(a.size, DUMP_MAX_ELEMENTS, replace=False))
            np.save(os.path.join(out_dir, f"{name}_sample.npy"), a[idx].astype(np.float32))
        else:
            np.save(os.path.join(out_dir, f"{name}.npy"), a.astype(np.float32))


def asg_point(tm: "Timed", rank, steps, warmup, profile=True, cfg=None, check=False):
    """fused ASG forward+backward at one (T, B) point; returns a dict of measurements."""
    import torch

    import wav2letter_b200 as w
    from wav2letter_b200 import capi

    cfg = dict(cfg or ASG_CFG)
    B, T, N, L = cfg["B"], cfg["T"], cfg["N"], cfg["L"]
    rng = np.random.default_rng(1234 + rank)
    nsets = cfg["n_input_sets"]
    host_e, host_y, dev_e, dev_y, np_sets = [], [], [], [], []
    tr_np = None
    for _ in range(nsets):
        e, tr_np, y = make_asg_inputs(rng, B, T, N, L)
        np_sets.append((e, y))
        he, hy = torch.from_numpy(e).pin_memory(), torch.from_numpy(y).pin_memory()
        host_e.append(he)
        host_y.append(hy)
        dev_e.append(he.to(tm.dev))
        dev_y.append(hy.to(tm.dev))
    trans = torch.from_numpy(tr_np).to(tm.dev)
    loss = torch.empty(B, dtype=torch.float32, device=tm.dev)
    d_emis = torch.empty((B, T, N), dtype=torch.float32, device=tm.dev)
    d_trans = torch.empty((N, N), dtype=torch.float32, device=tm.dev)
    ws = torch.empty(capi.lib.w2l_asg_workspace_size(B, T, N, L), dtype=torch.uint8, device=tm.dev)
    stage_e = torch.empty((B, T, N), dtype=torch.float32, device=tm.dev)
    stage_y = torch.empty((B, L), dtype=torch.int32, device=tm.dev)
    host_loss = torch.empty(B, dtype=torch.float32).pin_memory()

    def step(i):
        k = i % nsets
        w.asg_forward_backward(dev_e[k], dev_y[k], trans, cfg["scale_mode"], out=(loss, d_emis, d_trans), ws=ws)

    def step_e2e(i):
        k = i % nsets
        stage_e.copy_(host_e[k], non_blocking=True)
        stage_y.copy_(host_y[k], non_blocking=True)
        w.asg_forward_backward(stage_e, stage_y, trans, cfg["scale_mode"], out=(loss, d_emis, d_trans), ws=ws)
        host_loss.copy_(loss, non_blocking=True)

    parity = None
    if check:  # oracle parity of this very point (test infrastructure used as the checker)
        import oracle

        step(0)
        torch.cuda.synchronize()
        ol, ode, odt = oracle.asg(np_sets[0][0], np_sets[0][1], tr_np, cfg["scale_mode"])

        def rel(a, b):
            return float(np.abs(a - b).max() / max(1e-20, np.abs(b).max()))
        parity = {"loss": rel(loss.cpu().numpy(), ol), "d_emis": rel(d_emis.cpu().numpy(), ode), "d_trans": rel(d_trans.cpu().numpy(), odt)}
    prof = capi.ProfileList(2, 8) if profile else None
    ms, kern, launches, clocks = tm.run(step, steps, warmup, sample_clocks=profile, profile=prof, profile_steps=min(steps, 8))
    outputs = {"loss": loss.clone(), "d_emis": d_emis.clone(), "d_trans": d_trans.clone()}  # the last timed step's results
    ms_e2e, _, _, _ = tm.run(step_e2e, steps, warmup)
    kavg = sum(kern) / len(kern) if kern else None
    return dict(cfg=cfg, ms=ms / steps, ms_e2e=ms_e2e / steps, kernel_ms=kavg, launches=launches, clocks=clocks,
                ws_mb=ws.numel() / 1e6, h2d=B * T * N * 4 + B * L * 4, d2h=B * 4, parity=parity, outputs=outputs)


def run_asg(args, rank, world, local_rank):
    tm = Timed(world, local_rank)
    r = asg_point(tm, rank, args.steps, args.warmup, check=True)
    if rank != 0:
        return
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, r["outputs"])
    cfg = r["cfg"]
    B, T, N, L = cfg["B"], cfg["T"], cfg["N"], cfg["L"]
    peaks, src = measured_peaks()
    alg = asg_algorithmic_bytes(B, T, N, L)
    achieved = alg / (r["kernel_ms"] * 1e-3) / 1e9
    cpu_fps, cpu_s, cpu_threads = cpu_asg(B, cfg)
    traffic = None
    tp = os.path.join(ROOT, "profiles", "asg_chains_traffic.json")
    if os.path.exists(tp):
        traffic = json.load(open(tp)).get("dram_bytes_per_launch")
    frames = B * T * world
    line = {
        "metric": "frames_per_sec", "value": frames / (r["ms"] * 1e-3), "unit": "frames/s", "n_gpus": world, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": r["ms"], "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": "ASG criterion fwd+bwd, T=1500 N=30 B=64 L<=250 per GPU (BASELINE.json configs[4] point)",
                   "criterion": "asg", "scale_mode": cfg["scale_mode"], "sharding": f"utterances, dp{world}",
                   "cold_inputs": f"rotating {cfg['n_input_sets']} input sets ({cfg['n_input_sets'] * B * T * N * 4 / 1e6:.0f} MB) + "
                                  f"{r['ws_mb']:.0f} MB workspace rewritten per step > 50 MB L2"},
        "asg_fwd_bwd_ms_per_batch": r["ms"], "oracle_parity_rel": r["parity"],
        "clocks": r["clocks"],
        "e2e": {"value": frames / (r["ms_e2e"] * 1e-3), "unit": "frames/s", "ms_per_step": r["ms_e2e"],
                "h2d_bytes_per_step": r["h2d"], "d2h_bytes_per_step": r["d2h"]},
        "gpu_launches": r["launches"],
        "roofline": {"bound": "hbm", "kernel": "asg_chains_kernel", "achieved": achieved, "peak": peaks["hbm_gbs"],
                     "unit": "GB/s", "frac": achieved / peaks["hbm_gbs"], "traffic": traffic, "peak_source": src,
                     "kernel_ms": r["kernel_ms"], "algorithmic_bytes": alg, "dependent_step_ns": 1e6 * r["kernel_ms"] / T,
                     "note": "latency-bound recursion: T dependent steps per utterance; see DESIGN.md"},
        "cpu_baseline": {"value": cpu_fps, "unit": "frames/s", "cores": cpu_threads, "kind": "port",
                         "sample": f"1 batch B={B},T={T},N={N} (best of 3, {cpu_s:.2f} s)"},
    }
    print(json.dumps(line), flush=True)


def run_asg_sweep(args, rank, world, local_rank):
    """BASELINE.json configs[4]: T x B sweep (per-GPU batch; ranks run independent utterance shards), oracle parity on every point."""
    tm = Timed(world, local_rank)
    peaks, src = measured_peaks()
    points = []
    for T in (100, 500, 1500, 4000):
        for B in (1, 16, 64, 256):
            cfg = dict(T=T, N=30, B=B, L=max(2, T // 6), scale_mode="target_sz_sqrt", n_input_sets=max(2, min(16, (160 << 20) // (B * T * 120))))
            r = asg_point(tm, rank, args.steps, args.warmup, profile=True, cfg=cfg, check=(rank == 0))
            if rank == 0 and T == 1500 and B == 64 and args.dump_outputs:
                dump_outputs(args.dump_outputs, r["outputs"])
            alg = asg_algorithmic_bytes(B, T, 30, cfg["L"])
            if rank == 0:
                points.append({"T": T, "B": B, "L": cfg["L"], "ms_per_batch": r["ms"], "e2e_ms_per_batch": r["ms_e2e"],
                               "frames_per_sec": B * T * world / (r["ms"] * 1e-3), "chains_kernel_ms": r["kernel_ms"],
                               "algorithmic_GBps": alg / (r["ms"] * 1e-3) / 1e9, "hbm_frac": alg / (r["ms"] * 1e-3) / 1e9 / peaks["hbm_gbs"],
                               "dependent_step_ns": (1e6 * r["kernel_ms"] / T) if r["kernel_ms"] else None, "oracle_parity_rel": r["parity"]})
    if rank != 0:
        return
    worst = max(max(p["oracle_parity_rel"].values()) for p in points)
    head = next(p for p in points if p["T"] == 1500 and p["B"] == 64)
    line = {"metric": "frames_per_sec", "value": head["frames_per_sec"], "unit": "frames/s", "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": head["ms_per_batch"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic",
            "config": {"workload": "ASG criterion fwd+bwd sweep T in {100,500,1500,4000} x B in {1,16,64,256} per GPU, N=30 "
                                   "(BASELINE.json configs[4]); value = the T=1500,B=64 point", "sharding": f"utterances, dp{world}"},
            "worst_oracle_parity_rel": worst, "peak_source": src, "points": points}
    print(json.dumps(line), flush=True)


def run_train(args, rank, world, local_rank):
    import torch
    import torch.distributed as dist

    from wav2letter_b200 import capi
    from wav2letter_b200.trainer import Trainer, init_distributed, nccl_unique_id

    tm = Timed(world, local_rank)
    cfg = dict(WORKLOADS[args.workload])
    precision = cfg["precision"] if args.precision == "config" else args.precision
    B, T, F, N, L = cfg["B"], cfg["T"], cfg["F"], cfg["N"], cfg["L"]
    if world > 1:
        uid = torch.zeros(128, dtype=torch.uint8, device=tm.dev)
        if rank == 0:
            uid.copy_(torch.tensor(list(nccl_unique_id()), dtype=torch.uint8))
        dist.broadcast(uid, 0)
        init_distributed(rank, world, bytes(uid.cpu().tolist()))

    def make_trainer(c, prec):
        t = Trainer(c["arch"], c["F"], c["N"], c["crit"], c["scale_mode"], transdiag=c["transdiag"], lr=c["lr"], lrcrit=c["lrcrit"],
                    momentum=c["momentum"], maxgradnorm=c["maxgradnorm"], precision=prec)
        t.sync_parameters()  # fl::allReduceParameters at the start of train(), Train.cpp:1078-1079
        return t

    trainer = make_trainer(cfg, precision)
    rng = np.random.default_rng(1234 + rank)
    nsets = cfg["n_input_sets"]
    host_f, host_y, dev_f, dev_y = [], [], [], []
    for _ in range(nsets):
        f, y = make_train_inputs(rng, cfg)
        hf, hy = torch.from_numpy(f).pin_memory(), torch.from_numpy(y).pin_memory()
        host_f.append(hf)
        host_y.append(hy)
        dev_f.append(hf.to(tm.dev))
        dev_y.append(hy.to(tm.dev))
    loss = torch.empty(B, dtype=torch.float32, device=tm.dev)
    stage_f = torch.empty((B, 1, F, T), dtype=torch.float32, device=tm.dev)
    stage_y = torch.empty((B, L), dtype=torch.int32, device=tm.dev)
    host_loss = torch.empty(B, dtype=torch.float32).pin_memory()
    total_batch = float(B * world)

    def step(i, tr=None):
        k = i % nsets
        (tr or trainer).step(dev_f[k], dev_y[k], True, total_batch, loss)

    def step_e2e(i):
        k = i % nsets
        stage_f.copy_(host_f[k], non_blocking=True)
        stage_y.copy_(host_y[k], non_blocking=True)
        trainer.step(stage_f, stage_y, True, total_batch, loss)
        host_loss.copy_(loss, non_blocking=True)

    prof_steps = min(args.steps, 3)
    gemm_flops, t_out = arch_gemm_flops(cfg["arch"], B, T, F, N)
    prof = capi.ProfileList(1, 400 * prof_steps)
    ms, kern, launches, clocks = tm.run(step, args.steps, args.warmup, sample_clocks=True, profile=prof, profile_steps=prof_steps)
    if rank == 0 and args.dump_outputs:  # the last timed step's losses and the parameters it updated
        dump_outputs(args.dump_outputs, {"loss": loss, "params": trainer.get_flat(0)})
    ms_e2e, _, _, _ = tm.run(step_e2e, args.steps, args.warmup)
    final_loss = float(loss.sum().item())
    skipped = trainer.skipped_steps()
    # after the timed regions: one traced step (an event after every launch) -> warm in-situ share of each kernel
    tr = capi.trace(lambda: step(0))
    tr_total = sum(v[1] for v in tr.values()) or 1.0
    breakdown = {k: {"launches": v[0], "ms": round(v[1], 4), "share": round(v[1] / tr_total, 4)}
                 for k, v in sorted(tr.items(), key=lambda kv: -kv[1][1])}
    extras = {}
    if args.workload == "tds_ctc" and world == 1 and not args.no_extras:
        # the same step in the other precisions, the TDS+ASG step BASELINE.json's metric names, and the ASG point
        sweep = {precision: {"ms_per_step": ms / args.steps, "frames_per_sec": B * T * args.steps / (ms * 1e-3)}}
        for prec in ("f32", "tf32", "bf16"):
            if prec == precision:
                continue
            t2 = make_trainer(cfg, prec)
            k = args.steps
            ms2, _, _, _ = tm.run(lambda i: step(i, t2), k, args.warmup)
            sweep[prec] = {"ms_per_step": ms2 / k, "frames_per_sec": B * T * k / (ms2 * 1e-3)}
            t2.close()
        extras["precision_sweep"] = sweep
        c2 = dict(WORKLOADS["tds_asg"])
        t3 = make_trainer(c2, c2["precision"])
        f3, y3 = make_train_inputs(np.random.default_rng(77), c2)
        df3, dy3 = torch.from_numpy(f3).to(tm.dev), torch.from_numpy(y3).to(tm.dev)
        l3 = torch.empty(c2["B"], dtype=torch.float32, device=tm.dev)
        k = args.steps
        ms3, _, _, _ = tm.run(lambda i: t3.step(df3, dy3, True, float(c2["B"]), l3), k, args.warmup)
        extras["tds_asg_point"] = {"workload": train_workload_text(c2), "precision": c2["precision"], "ms_per_step": ms3 / k,
                                   "frames_per_sec_per_gpu": c2["B"] * c2["T"] * k / (ms3 * 1e-3), "final_loss_sum": float(l3.sum().item())}
        t3.close()
        asg = asg_point(tm, rank, args.steps, args.warmup, profile=False)
        alg = asg_algorithmic_bytes(ASG_CFG["B"], ASG_CFG["T"], ASG_CFG["N"], ASG_CFG["L"])
        extras["asg_fwd_bwd_ms_per_batch"] = asg["ms"]
        extras["asg_point"] = {"config": "T=1500 N=30 B=64", "ms_per_batch": asg["ms"], "e2e_ms_per_batch": asg["ms_e2e"],
                               "frames_per_sec": ASG_CFG["B"] * ASG_CFG["T"] / (asg["ms"] * 1e-3), "algorithmic_GBps": alg / (asg["ms"] * 1e-3) / 1e9}
    if rank != 0:
        return
    peaks, src = measured_peaks()
    frames = B * T * world
    gemm_ms_per_step = sum(kern) / max(1, prof_steps)
    achieved = gemm_flops / (gemm_ms_per_step * 1e-3) / 1e12
    peak = peaks.get("bf16_tflops_sustained", peaks["bf16_tflops"])
    cpu = None
    if world == 1 and not args.no_cpu:  # CPU baseline: rank 0 at N=1 only, bounded sample
        r = CpuArm(cfg).run(2, 1, budget_s=25.0)
        cpu = {"value": r["fps"], "unit": "frames/s", "cores": r["threads"], "kind": "port",
               "sample": f"2 train steps of B={r['B']},T={T} on torch-CPU/oneDNN fp32 + C-oracle {cfg['crit'].upper()} ({r['s_per_step']:.1f} s/step)"}
    traffic = None
    tp = os.path.join(ROOT, "profiles", "gemm_traffic.json")
    if os.path.exists(tp):
        traffic = json.load(open(tp)).get(f"dram_bytes_per_launch_{precision}")
    kname = {"f32": "gemm_wgmma_kernel<f32x3>", "tf32": "gemm_wgmma_kernel<tf32>", "bf16": "gemm_wgmma_kernel<bf16>"}[precision]
    line = {
        "metric": "frames_per_sec", "value": frames * args.steps / (ms * 1e-3), "unit": "frames/s", "n_gpus": world,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": precision, "dtype_note": DTYPE_NOTE[precision], "data": "synthetic",
        "config": {"workload": train_workload_text(cfg), "global_batch": B * world, "frames_per_utterance": T, "output_frames": t_out,
                   "parallelism": f"dp{world}", "precision": precision,
                   "optimizer": f"SGD lr={cfg['lr']} lrcrit={cfg['lrcrit']} momentum={cfg['momentum']} maxgradnorm={cfg['maxgradnorm']}",
                   "dropout": "as in the arch file", "params": trainer.num_params(0),
                   "cold_inputs": f"rotating {nsets} input sets; activations + gradients of a step ({B}x{T} frames) exceed the 50 MB L2"},
        "final_loss_sum": final_loss, "skipped_steps_nan_guard": skipped,
        "clocks": clocks,
        "e2e": {"value": frames * args.steps / (ms_e2e * 1e-3), "unit": "frames/s", "ms_per_step": ms_e2e / args.steps,
                "h2d_bytes_per_step": B * F * T * 4 + B * L * 4, "d2h_bytes_per_step": B * 4},
        "gpu_launches": launches,
        "roofline": {"bound": "tensor", "kernel": kname, "achieved": achieved, "peak": peak, "unit": "TFLOP/s",
                     "frac": achieved / peak, "traffic": traffic,
                     "peak_source": src + "; peak = bf16 (tf32 / f32x3 math has 1/2 / 1/6 of the bf16 hardware ceiling)",
                     "gemm_ms_per_step": gemm_ms_per_step, "gemm_launches_per_step": len(kern) / max(1, prof_steps),
                     "algorithmic_flops_per_step": gemm_flops, "gemm_share_of_step": gemm_ms_per_step / (ms / args.steps),
                     "gemm_launch_us_first_step": [round(1e3 * t, 1) for t in kern[:int(len(kern) / max(1, prof_steps))]]},
        "step_breakdown": {"method": "one extra traced step after the timed region, a CUDA event after every launch",
                           "traced_ms": round(tr_total, 3), "kernels": dict(list(breakdown.items())[:16])},
        "cpu_baseline": cpu,
    }
    line.update(extras)
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--workload", default="tds_ctc", choices=["tds_ctc", "tds_asg", "conv_glu_asg", "streaming_tds_ctc", "asg", "asg_sweep"])
    ap.add_argument("--precision", default="config", choices=["config", "f32", "tf32", "bf16"])
    ap.add_argument("--no-extras", action="store_true", help="skip the precision sweep / TDS+ASG / ASG point of the default workload")
    ap.add_argument("--no-cpu", action="store_true", help="skip the CPU baseline leg")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the timed path computed in its last step to DIR/<name>.npy")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if args.impl == "reference":
        run_reference(args, rank, world)
        return
    args.warmup = max(args.warmup, 3)
    import torch

    torch.cuda.set_device(local_rank)
    if world > 1:
        import torch.distributed as dist

        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    try:
        fn = {"asg": run_asg, "asg_sweep": run_asg_sweep}.get(args.workload, run_train)
        fn(args, rank, world, local_rank)
    finally:
        if world > 1:
            import torch.distributed as dist

            dist.destroy_process_group()


if __name__ == "__main__":
    main()
