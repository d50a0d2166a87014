"""Kernel-level diagnosis of the fp32-accurate mode at the small stage-3 sizes of the arch parity test (T' = 20 frames)."""
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import wav2letter_b200 as w  # noqa: E402
from wav2letter_b200 import capi  # noqa: E402

out = {}


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / max(1e-12, float(b.double().abs().max())))


# ---- GEMM: wgrad with a short K, dgrad with mask + accumulate ------------------------------------------
for kind in ("tf32", "f32x3"):
    for (M, N, K) in [(1440, 1440, 40), (1120, 1120, 80), (800, 800, 160), (2000, 1440, 40)]:
        A = torch.randn(K, M, device="cuda")
        B = torch.randn(K, N, device="cuda")
        C = capi.gemm(A, B, kind, True, True)
        ref = A.double().t() @ B.double()
        out[f"gemm_wgrad_{kind}_{M}x{N}x{K}"] = rel(C, ref)
        C0 = torch.randn(M, N, device="cuda")
        C2 = C0.clone()
        capi.gemm(A, B, kind, True, True, out=C2, accumulate=True)
        out[f"gemm_wgrad_acc_{kind}_{M}x{N}x{K}"] = rel(C2, ref + C0.double())
    M, N, K = 40, 1440, 1440
    A = torch.randn(M, K, device="cuda")
    B = torch.randn(K, N, device="cuda")
    aux = torch.randn(M, N, device="cuda")
    C0 = torch.randn(M, N, device="cuda")
    C2 = C0.clone()
    capi.gemm(A, B, kind, False, True, out=C2, accumulate=True, aux=aux, aux_mode=1, aux_scale=1.0)
    out[f"gemm_dgrad_mask_acc_{kind}"] = rel(C2, C0.double() + (A.double() @ B.double()) * (aux > 0))
    Bw = torch.randn(N, K, device="cuda")
    bias = torch.randn(N, device="cuda")
    Y = capi.gemm(A, Bw, kind, False, False, bias=bias, act=1)
    out[f"gemm_fwd_bias_relu_{kind}"] = rel(Y, (A.double() @ Bw.double().t() + bias.double()).clamp_min(0))

# ---- LayerNorm whole-sample forward / backward -----------------------------------------------------------
for (B_, R) in [(2, 20 * 1440), (2, 40 * 1120), (2, 80 * 800), (16, 150 * 1440)]:
    a = torch.randn(B_, R, device="cuda")
    r = torch.randn(B_, R, device="cuda")
    g = torch.tensor([1.3], device="cuda")
    bb = torch.tensor([0.2], device="cuda")
    y, mr = capi.layernorm_fwd(a, r, g, bb)
    a64, r64 = a.double().requires_grad_(True), r.double().requires_grad_(True)
    g64, b64 = g.double().requires_grad_(True), bb.double().requires_grad_(True)
    yr = F.layer_norm(a64 + r64, (R,), eps=1e-5) * g64 + b64
    out[f"ln_fwd_{B_}x{R}"] = rel(y, yr)
    dy = torch.randn(B_, R, device="cuda")
    yr.backward(dy.double())
    d_branch, d_res, dgain, dbias = capi.layernorm_bwd(a, r, dy, g, mr, 1, 1.0)
    out[f"ln_bwd_dres_{B_}x{R}"] = rel(d_res, r64.grad)
    out[f"ln_bwd_dbranch_{B_}x{R}"] = rel(d_branch, a64.grad * (a64 > 0))
    out[f"ln_bwd_dgain_{B_}x{R}"] = rel(dgain, g64.grad)
    out[f"ln_bwd_dbias_{B_}x{R}"] = rel(dbias, b64.grad)


# ---- time convolution at T < kernel ----------------------------------------------------------------------
def ref_conv(x, wt, bias, stride, pad_left, Tout):
    B, T, Cin, W = x.shape
    K = wt.shape[2]
    xin = x.permute(0, 2, 1, 3)
    need = (Tout - 1) * stride + K
    pr = max(0, need - T - pad_left)
    y = F.conv2d(F.pad(xin, (0, 0, pad_left, pr)), wt.unsqueeze(-1), bias, stride=(stride, 1))
    return y[:, :, :Tout].permute(0, 2, 1, 3).contiguous()


for (B_, T, C, K, pl) in [(2, 20, 18, 21, 10), (2, 40, 14, 21, 10), (2, 80, 10, 21, 10), (2, 20, 27, 11, 10), (2, 5, 18, 21, 10)]:
    x = torch.randn(B_, T, C, 80, device="cuda")
    wt = torch.randn(C, C, K, device="cuda") * 0.1
    bias = torch.randn(C, device="cuda")
    Tout = T if pl * 2 == K - 1 else T
    x64, w64, b64 = x.double().requires_grad_(True), wt.double().requires_grad_(True), bias.double().requires_grad_(True)
    pre = ref_conv(x64, w64, b64, 1, pl, Tout)
    dy = torch.randn(B_, Tout, C, 80, device="cuda")
    pre.backward(dy.double())
    for path, prec in [("mma", "tf32"), ("x3", "f32")]:
        try:
            capi.set_precision(prec)
            y = capi.conv_time_fwd(x, wt, bias, Tout, 1, pl)
            dx = capi.conv_time_dgrad(dy, wt, T, 1, pl)
            dwt, dbias = capi.conv_time_wgrad(x, dy, K, 1, pl)
            out[f"conv_{path}_T{T}_C{C}_K{K}"] = [rel(y, pre), rel(dx, x64.grad), rel(dwt, w64.grad), rel(dbias, b64.grad)]
        except Exception as e:  # noqa: BLE001
            out[f"conv_{path}_T{T}_C{C}_K{K}"] = "ERR " + str(e)[:100]
        finally:
            capi.set_precision("tf32")

for k, v in out.items():
    print(k, v)
json.dump(out, sys.stdout, indent=1)
