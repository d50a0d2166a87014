"""GPU parity of the acoustic-model kernels (time convolution fwd/dgrad/wgrad, per-sample LayerNorm with
fused residual, dropout, extended GEMM epilogue, flat-arena SGD) against torch float64 references of the
same ops, plus the reference's own Conv1d known-answer vector."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / max(1e-6, float(b.double().abs().max())))


def ref_conv(x, wt, bias, stride, pad_left, Tout):
    """x [B,T,Cin,W] f64, wt [Cout,Cin,K]: out[b,to,co,w] = sum x[b,to*s+dk-pl,ci,w] wt[co,ci,dk] + bias"""
    B, T, Cin, W = x.shape
    K = wt.shape[2]
    xin = x.permute(0, 2, 1, 3)  # [B,Cin,T,W]
    need = (Tout - 1) * stride + K
    pad_right = max(0, need - T - pad_left)
    xin = F.pad(xin, (0, 0, pad_left, pad_right))
    y = F.conv2d(xin, wt.unsqueeze(-1), bias, stride=(stride, 1))
    return y[:, :, :Tout].permute(0, 2, 1, 3).contiguous()


@pytest.mark.parametrize("B,T,Cin,Cout,K,stride,W", [
    (2, 37, 10, 10, 21, 1, 80), (3, 50, 1, 10, 21, 2, 80), (2, 41, 10, 14, 21, 2, 80), (2, 33, 18, 18, 21, 1, 80),
    (1, 20, 27, 27, 11, 1, 80), (2, 9, 3, 5, 3, 1, 7), (2, 30, 15, 19, 10, 2, 80), (1, 3, 10, 10, 21, 1, 80),
])
def test_conv_time_fwd_dgrad_wgrad(B, T, Cin, Cout, K, stride, W):
    from wav2letter_b200 import capi

    g = torch.Generator(device="cuda").manual_seed(B * 100 + T)
    x = torch.randn((B, T, Cin, W), device="cuda", generator=g)
    wt = torch.randn((Cout, Cin, K), device="cuda", generator=g) * 0.1
    bias = torch.randn(Cout, device="cuda", generator=g)
    # flashlight SAME padding (symmetric): p = ceil(((K-1) - (T % s or s) + 1) / 2)
    rem = T % stride
    tot = (K - 1) - (stride if rem == 0 else rem) + 1
    pl = max((tot + 1) // 2, 0)
    Tout = (T + 2 * pl - K) // stride + 1
    add = torch.randn((B, Tout, Cout, W), device="cuda", generator=g)
    y = capi.conv_time_fwd(x, wt, bias, Tout, stride, pl, act=1, add=add)
    x64 = x.double().requires_grad_(True)
    w64 = wt.double().requires_grad_(True)
    b64 = bias.double().requires_grad_(True)
    pre = ref_conv(x64, w64, b64, stride, pl, Tout)
    yr = pre.clamp_min(0) + add.double()
    # W % 8 == 0 routes to the tensor-core path (mma.sync TF32 operands, fp32 accumulate): TF32 tolerance;
    # other widths use the fp32 SIMT kernels
    tol = 3e-3 if W % 8 == 0 else 1e-5
    assert rel(y, yr) < tol
    dy = torch.randn((B, Tout, Cout, W), device="cuda", generator=g)
    pre.backward(dy.double())
    addx = torch.randn((B, T, Cin, W), device="cuda", generator=g)
    dx = capi.conv_time_dgrad(dy, wt, T, stride, pl, add=addx)
    assert rel(dx, x64.grad + addx.double()) < tol
    inplace = addx.clone()  # add == dx: the residual gradient is accumulated in place (fl_compat's autograd does this)
    capi.conv_time_dgrad(dy, wt, T, stride, pl, add=inplace, out=inplace)
    assert torch.equal(inplace, dx)
    dwt, dbias = capi.conv_time_wgrad(x, dy, K, stride, pl)
    assert rel(dwt, w64.grad) < tol
    assert rel(dbias, b64.grad) < tol


def test_conv1d_reference_golden():
    """Conv1dTest.cpp:32-104 — tolerance 1e-2 there (fp16-packed weights); we are exact fp32."""
    import conv1d_reference_golden as G
    from wav2letter_b200 import capi

    inp = torch.tensor(G.INPUT, dtype=torch.float32).view(G.T, G.GROUPS, G.CH_PER_GROUP)
    tgt = torch.tensor(G.TARGET, dtype=torch.float32).view(G.T, G.GROUPS, G.CH_PER_GROUP)
    wt = torch.tensor(G.WEIGHTS, dtype=torch.float32).view(G.CH_PER_GROUP, G.KW, G.CH_PER_GROUP)  # [co][dk][ci]
    x = inp.permute(0, 2, 1).unsqueeze(0).contiguous().cuda()  # [1,T,C=2,W=groups]
    w = wt.permute(0, 2, 1).contiguous().cuda()                # [co][ci][dk]
    y = capi.conv_time_fwd(x, w, torch.tensor(G.BIAS).cuda(), G.T, 1, G.PAD)
    out = y[0].permute(0, 2, 1).cpu()  # [T][groups][c]
    assert float((out - tgt).abs().max()) < 1e-2


def test_dropout_in_conv_and_gemm():
    from wav2letter_b200 import capi

    x = torch.ones((2, 64, 4, 80), device="cuda")
    wt = torch.zeros((4, 4, 1), device="cuda")
    for c in range(4):
        wt[c, c, 0] = 1.0
    y = capi.conv_time_fwd(x, wt, None, 64, 1, 0, dropout_p=0.2, seed=7)
    kept = (y != 0).float().mean().item()
    assert abs(kept - 0.8) < 0.01
    assert torch.allclose(y[y != 0], torch.tensor(1.25, device="cuda"))
    y2 = capi.conv_time_fwd(x, wt, None, 64, 1, 0, dropout_p=0.2, seed=7)
    y3 = capi.conv_time_fwd(x, wt, None, 64, 1, 0, dropout_p=0.2, seed=8)
    assert torch.equal(y, y2) and not torch.equal(y, y3)
    A = torch.ones((256, 32), device="cuda")
    Bm = torch.ones((384, 32), device="cuda")
    out = torch.empty((256, 384), device="cuda")
    capi.gemm_tf32_ex(A, Bm, out, dropout_p=0.5, seed=3)
    kept = (out != 0).float().mean().item()
    assert abs(kept - 0.5) < 0.01 and torch.allclose(out[out != 0], torch.tensor(64.0, device="cuda"))


@pytest.mark.parametrize("B,R", [(1, 17), (3, 5000), (4, 50 * 800), (2, 250 * 1440),
                                 (2400, 1200), (1500, 2160), (1300, 30)])  # many short groups: the one-warp-per-group kernels
def test_layernorm_fwd_bwd(B, R):
    from wav2letter_b200 import capi

    g = torch.Generator(device="cuda").manual_seed(R)
    a = torch.randn((B, R), device="cuda", generator=g).clamp_min(0) * 1.3   # branch output (post ReLU: has zeros)
    r = torch.randn((B, R), device="cuda", generator=g) * 2 + 0.5
    gain = torch.tensor([1.7], device="cuda")
    bias = torch.tensor([-0.3], device="cuda")
    y, mr = capi.layernorm_fwd(a, r, gain, bias)
    a64, r64 = a.double().requires_grad_(True), r.double().requires_grad_(True)
    g64, b64 = gain.double().requires_grad_(True), bias.double().requires_grad_(True)
    yr = F.layer_norm(a64 + r64, (R,), eps=1e-5) * g64 + b64
    assert rel(y, yr) < 1e-5
    dy = torch.randn((B, R), device="cuda", generator=g)
    yr.backward(dy.double())
    d_branch, d_res, dgain, dbias = capi.layernorm_bwd(a, r, dy, gain, mr, branch_mode=1, branch_scale=1.25)
    assert rel(d_res, r64.grad) < 2e-5
    assert rel(d_branch, a64.grad * (a.double() > 0) * 1.25) < 2e-5
    assert rel(dgain, g64.grad) < 1e-4 and rel(dbias, b64.grad) < 1e-4
    d_b2, _, _, _ = capi.layernorm_bwd(a, r, dy, gain, mr, branch_mode=2, branch_scale=2.0)
    assert rel(d_b2, a64.grad * (a.double() != 0) * 2.0) < 2e-5


def test_gemm_epilogue_mask_and_accumulate():
    from wav2letter_b200 import capi

    g = torch.Generator(device="cuda").manual_seed(5)
    A = torch.randn((300, 64), device="cuda", generator=g)
    Bm = torch.randn((200, 64), device="cuda", generator=g)
    aux = torch.randn((300, 200), device="cuda", generator=g).clamp_min(0)
    C0 = torch.randn((300, 200), device="cuda", generator=g)
    out = C0.clone()
    capi.gemm_tf32_ex(A, Bm, out, accumulate=True, aux=aux, aux_mode=1, aux_scale=1.25)
    ref = C0.double() + (A.double() @ Bm.double().t()) * (aux.double() > 0) * 1.25
    assert rel(out, ref) < 2e-3


def test_colsum_sqnorm_sgd():
    from wav2letter_b200 import capi
    import ctypes

    g = torch.Generator(device="cuda").manual_seed(9)
    X = torch.randn((1000, 77), device="cuda", generator=g)
    out = torch.ones(77, device="cuda")
    capi._check(capi.lib.w2l_colsum_accumulate(capi._stream(), 1000, 77, capi._ptr(X), 77, capi._ptr(out)))
    assert rel(out, 1 + X.double().sum(0)) < 1e-5
    X4 = torch.randn((2403, 1120), device="cuda", generator=g)   # float4 path (N % 4 == 0), sub-matrix with ld > N
    out4 = torch.ones(1000, device="cuda")
    capi._check(capi.lib.w2l_colsum_accumulate(capi._stream(), 2403, 1000, capi._ptr(X4), 1120, capi._ptr(out4)))
    assert rel(out4, 1 + X4[:, :1000].double().sum(0)) < 1e-5
    n = 100003
    p = torch.randn(n, device="cuda", generator=g)
    gr = torch.randn(n, device="cuda", generator=g)
    v = torch.randn(n, device="cuda", generator=g)
    sq = torch.zeros(1, dtype=torch.float64, device="cuda")
    capi._check(capi.lib.w2l_sq_norm_accumulate(capi._stream(), n, capi._ptr(gr), capi._ptr(sq)))
    assert abs(sq.item() - float((gr.double() ** 2).sum())) < 1e-6 * sq.item()
    lr, mom, wd, gs, mx = 0.1, 0.9, 1e-3, 0.25, 1.0
    p0, v0 = p.double().clone(), v.double().clone()
    capi._check(capi.lib.w2l_sgd_step(capi._stream(), n, capi._ptr(p), capi._ptr(gr), capi._ptr(v), lr, mom, wd, gs, mx,
                                      capi._ptr(sq)))
    nrm = float(sq.item()) ** 0.5 * gs
    scale = gs * (mx / (nrm + 1e-6) if nrm > mx else 1.0)
    ge = gr.double() * scale + wd * p0
    ve = mom * v0 + ge
    assert rel(v, ve) < 1e-5 and rel(p, p0 - lr * ve) < 1e-5


@pytest.mark.parametrize("path", ["tf32", "mma", "x3", "simt"])
@pytest.mark.parametrize("B,T,Cin,Cout,K,stride,pl,pr", [
    (2, 40, 23, 23, 11, 1, 10, 0), (2, 40, 15, 15, 9, 1, 7, 1), (2, 46, 19, 23, 12, 2, 9, 1), (2, 40, 23, 27, 11, 1, 10, 0),
    (2, 52, 1, 15, 10, 2, 5, 3), (2, 36, 27, 27, 11, 1, 10, 0), (1, 24, 18, 18, 21, 1, 10, 10),
])
def test_conv_time_streaming_shapes_all_paths(B, T, Cin, Cout, K, stride, pl, pr, path):
    """the asymmetric paddings of the streaming TDS arch (PD l r + C2, TDS with rightPadding) on the three arithmetic paths:
    the wgmma / TMA kernel (forward, stride-1 data gradient), the mma.sync TF32 kernels, the same in error-compensated
    3xTF32 (W2L_PRECISION_F32), and the fp32 SIMT fallback"""
    from wav2letter_b200 import capi

    W = 80
    g = torch.Generator(device="cuda").manual_seed(T * 7 + Cin)
    x = torch.randn((B, T, Cin, W), device="cuda", generator=g)
    wt = torch.randn((Cout, Cin, K), device="cuda", generator=g) * 0.1
    bias = torch.randn(Cout, device="cuda", generator=g)
    Tout = (T + pl + pr - K) // stride + 1
    x64, w64, b64 = x.double().requires_grad_(True), wt.double().requires_grad_(True), bias.double().requires_grad_(True)
    pre = ref_conv(x64, w64, b64, stride, pl, Tout)
    dy = torch.randn((B, Tout, Cout, W), device="cuda", generator=g)
    pre.backward(dy.double())
    try:
        capi.set_precision("f32" if path == "x3" else "tf32")
        capi._check(capi.lib.w2l_conv_set_path({"simt": 1, "mma": 2, "tf32": 3}.get(path, 0)))  # "tf32" = the wgmma kernel
        y = capi.conv_time_fwd(x, wt, bias, Tout, stride, pl)
        dx = capi.conv_time_dgrad(dy, wt, T, stride, pl)
        dwt, dbias = capi.conv_time_wgrad(x, dy, K, stride, pl)
    finally:
        capi.set_precision("tf32")
        capi._check(capi.lib.w2l_conv_set_path(0))
    tol = 3e-3 if path in ("tf32", "mma") else 2e-5
    assert rel(y, pre) < tol, (path, rel(y, pre))
    assert rel(dx, x64.grad) < tol, (path, rel(dx, x64.grad))
    assert rel(dwt, w64.grad) < tol, (path, rel(dwt, w64.grad))
    assert rel(dbias, b64.grad) < tol


def test_conv_time_wgmma_path_falls_back_when_the_window_does_not_fit():
    """w2l_conv_set_path(3) selects the wgmma kernel only where its window and weights fit in shared memory: at 32 channels
    and kw = 27 they do not (and the mma.sync kernel does not cover kw * C > 512), so the call runs on the SIMT kernels"""
    from wav2letter_b200 import capi

    B, T, C, K, pl, W = 1, 40, 32, 27, 13, 80
    g = torch.Generator(device="cuda").manual_seed(27)
    x = torch.randn((B, T, C, W), device="cuda", generator=g)
    wt = torch.randn((C, C, K), device="cuda", generator=g) * 0.1
    bias = torch.randn(C, device="cuda", generator=g)
    Tout = T + 2 * pl - K + 1
    x64, w64, b64 = x.double().requires_grad_(True), wt.double().requires_grad_(True), bias.double().requires_grad_(True)
    pre = ref_conv(x64, w64, b64, 1, pl, Tout)
    dy = torch.randn((B, Tout, C, W), device="cuda", generator=g)
    pre.backward(dy.double())
    try:
        capi._check(capi.lib.w2l_conv_set_path(3))
        y = capi.conv_time_fwd(x, wt, bias, Tout, 1, pl)
        dx = capi.conv_time_dgrad(dy, wt, T, 1, pl)
    finally:
        capi._check(capi.lib.w2l_conv_set_path(0))
    assert rel(y, pre) < 3e-3 and rel(dx, x64.grad) < 3e-3
