"""BASELINE.json metric (i): fused ASG forward+backward over T in {100,500,1500,4000} x B in {1,16,64,256}, N = 30.
Prints one line per point: ms/batch (CUDA events, rotating cold inputs), frames/s, algorithmic GB/s (SURVEY 8d bytes),
ns per dependent step, and the parity of the point against the CPU oracle where that finishes quickly."""
import json, os, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import wav2letter_b200 as w
from wav2letter_b200 import capi
from bench import make_asg_inputs, asg_algorithmic_bytes
import oracle

N = 30
rows = []
for T in (100, 500, 1500, 4000):
    for B in (1, 16, 64, 256):
        L = max(1, T // 6)
        rng = np.random.default_rng(1234)
        nsets = 4 if B * T * N * 4 * 4 < (1 << 30) else 2
        sets = []
        for _ in range(nsets):
            e, tr_np, y = make_asg_inputs(rng, B, T, N, L)
            sets.append((torch.from_numpy(e).cuda(), torch.from_numpy(y).cuda()))
        trans = torch.from_numpy(tr_np).cuda()
        loss = torch.empty(B, device="cuda"); de = torch.empty((B, T, N), device="cuda"); dt = torch.empty((N, N), device="cuda")
        ws = torch.empty(capi.lib.w2l_asg_workspace_size(B, T, N, L), dtype=torch.uint8, device="cuda")
        step = lambda i: w.asg_forward_backward(sets[i % nsets][0], sets[i % nsets][1], trans, "target_sz_sqrt", out=(loss, de, dt), ws=ws)
        for i in range(3):
            step(i)
        torch.cuda.synchronize()
        n = 20
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(n):
            step(i)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        err = None
        if B * T <= 16 * 1500:  # oracle check of the last computed set
            k = (n - 1) % nsets
            ol, ode, odt = oracle.asg(sets[k][0].cpu().numpy(), sets[k][1].cpu().numpy(), tr_np, "target_sz_sqrt")
            den = max(1e-6, float(np.abs(ode).max()))
            err = max(float(np.abs(loss.cpu().numpy() - ol).max() / max(1e-6, np.abs(ol).max())), float(np.abs(de.cpu().numpy() - ode).max() / den))
        alg = asg_algorithmic_bytes(B, T, N, L)
        row = dict(T=T, B=B, L=L, ms_per_batch=round(ms, 4), frames_per_s=round(B * T / ms * 1e3), alg_GBps=round(alg / ms / 1e6, 2),
                   ns_per_dependent_step=round(ms * 1e6 / T, 1), rel_err_vs_oracle=err)
        rows.append(row)
        print(json.dumps(row), flush=True)
