"""The float4 (V = 4) and scalar (V = 1) instances of the memory-bound passes that the other kernel tests do not reach:
WeightNorm at a row length that is a multiple of 4, and the LayerNorm backward on buffers that start one float into their
allocation (which forces V = 1).  Both against float64 torch, with the tolerances of test_gpu_am_kernels.py and
test_gpu_convglu.py.  GLU and axpy add in the same order at both widths, so their two instances must agree bit for bit."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def rel(a, b):
    a, b = a.detach(), b.detach()
    return float((a.double() - b.double()).abs().max() / max(1e-6, float(b.double().abs().max())))


def shifted(t, off):
    """a copy of t that starts `off` floats into its allocation"""
    buf = torch.empty(t.numel() + off, device=t.device, dtype=t.dtype)
    out = buf[off:].view(t.shape)
    out.copy_(t)
    return out


def test_weightnorm_float4_rows():
    from wav2letter_b200 import capi

    g = torch.Generator(device="cuda").manual_seed(4)
    rows, ln = 37, 528
    v = torch.randn(rows, ln, device="cuda", generator=g)
    gg = torch.rand(rows, device="cuda", generator=g) + 0.5
    w, inv = torch.empty_like(v), torch.empty(rows, device="cuda")
    capi._check(capi.lib.w2l_weightnorm_fwd(capi._stream(), rows, ln, capi._ptr(v), capi._ptr(gg), capi._ptr(w), capi._ptr(inv)))
    v64, g64 = v.double().requires_grad_(True), gg.double().requires_grad_(True)
    wr = g64[:, None] * v64 / v64.norm(dim=1, keepdim=True)
    assert rel(w, wr) < 1e-5
    dw = torch.randn(rows, ln, device="cuda", generator=g)
    wr.backward(dw.double())
    dv, dg = torch.zeros_like(v), torch.zeros_like(gg)
    capi._check(capi.lib.w2l_weightnorm_bwd(capi._stream(), rows, ln, capi._ptr(v), capi._ptr(gg), capi._ptr(inv), capi._ptr(dw),
                                            capi._ptr(dv), capi._ptr(dg)))
    assert rel(dv, v64.grad) < 1e-4 and rel(dg, g64.grad) < 1e-4


@pytest.mark.parametrize("B,R", [(3, 5000), (4, 50 * 800), (2400, 1200)])  # two-pass and one-warp-per-group kernels
def test_layernorm_bwd_scalar_chunks(B, R):
    from wav2letter_b200 import capi

    g = torch.Generator(device="cuda").manual_seed(R + 1)
    a = shifted(torch.randn((B, R), device="cuda", generator=g).clamp_min(0) * 1.3, 1)
    r = shifted(torch.randn((B, R), device="cuda", generator=g) * 2 + 0.5, 1)
    dy = shifted(torch.randn((B, R), device="cuda", generator=g), 1)
    gain = torch.tensor([1.7], device="cuda")
    bias = torch.tensor([-0.3], device="cuda")
    y, mr = capi.layernorm_fwd(a, r, gain, bias)
    a64, r64 = a.double().requires_grad_(True), r.double().requires_grad_(True)
    g64, b64 = gain.double().requires_grad_(True), bias.double().requires_grad_(True)
    yr = F.layer_norm(a64 + r64, (R,), eps=1e-5) * g64 + b64
    assert rel(y, yr) < 1e-5
    yr.backward(dy.double())
    d_branch, d_res = shifted(torch.zeros((B, R), device="cuda"), 1), shifted(torch.zeros((B, R), device="cuda"), 1)
    dgain, dbias = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    scratch = capi.layernorm_scratch(B, "cuda")
    capi._check(capi.lib.w2l_layernorm_bwd(capi._stream(), B, R, capi._ptr(a), capi._ptr(r), capi._ptr(dy), capi._ptr(gain), capi._ptr(mr),
                                           capi._ptr(d_branch), capi._ptr(d_res), 1, 1.25, capi._ptr(dgain), capi._ptr(dbias),
                                           capi._ptr(scratch)))
    assert rel(d_res, r64.grad) < 2e-5
    assert rel(d_branch, a64.grad * (a.double() > 0) * 1.25) < 2e-5
    assert rel(dgain, g64.grad) < 1e-4 and rel(dbias, b64.grad) < 1e-4


@pytest.mark.parametrize("p", [0.0, 0.3])
def test_glu_widths_agree(p):
    from wav2letter_b200 import capi

    g = torch.Generator(device="cuda").manual_seed(12)
    R, H = 501, 120
    x = torch.randn(R, 2 * H, device="cuda", generator=g)
    dy = torch.randn(R, H, device="cuda", generator=g)
    outs = []
    for off in (0, 1):
        xs, dys = shifted(x, off), shifted(dy, off)
        y, dx = shifted(torch.zeros(R, H, device="cuda"), off), shifted(torch.zeros(R, 2 * H, device="cuda"), off)
        capi._check(capi.lib.w2l_glu_fwd(capi._stream(), R, H, capi._ptr(xs), capi._ptr(y), p, 21))
        capi._check(capi.lib.w2l_glu_bwd(capi._stream(), R, H, capi._ptr(xs), capi._ptr(dys), capi._ptr(dx), p, 21))
        outs.append((y, dx))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


def test_axpy_widths_agree():
    from wav2letter_b200 import capi

    g = torch.Generator(device="cuda").manual_seed(13)
    n = 100000
    x = torch.randn(n, device="cuda", generator=g)
    y = torch.randn(n, device="cuda", generator=g)
    outs = []
    for off in (0, 1):
        xs, ys = shifted(x, off), shifted(y, off)
        capi._check(capi.lib.w2l_axpy(capi._stream(), n, 0.37, capi._ptr(xs), capi._ptr(ys)))
        outs.append(ys)
    assert torch.equal(outs[0], outs[1])
    assert rel(outs[0], y.double() + 0.37 * x.double()) < 1e-6
