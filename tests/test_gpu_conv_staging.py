"""The tensor-core time convolution's frame windows, against float64 references: windows at the ends of a sample, one
output frame, long samples (a weight-gradient CTA walks many chunks), the polyphase data gradient of stride-2
convolutions with odd T, narrow and wide column slices, and samples whose magnitudes differ by orders of magnitude (a
window that reads the neighbouring sample's frames shows up per sample).  Forward, data gradient and weight gradient,
in f32 (3xTF32) and tf32."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = {"f32": 2e-5, "tf32": 3e-3}


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / max(1e-30, float(b.abs().max())))


def ref_conv(x, wt, bias, stride, pad_left, Tout):
    """x [B,T,Cin,W] f64, wt [Cout,Cin,K]: out[b,to,co,w] = sum x[b,to*s+dk-pl,ci,w] wt[co,ci,dk] + bias"""
    B, T, Cin, W = x.shape
    K = wt.shape[2]
    need = (Tout - 1) * stride + K
    xin = F.pad(x.permute(0, 2, 1, 3), (0, 0, pad_left, max(0, need - T - pad_left)))
    return F.conv2d(xin, wt.unsqueeze(-1), bias, stride=(stride, 1))[:, :, :Tout].permute(0, 2, 1, 3).contiguous()


def run(prec, x, wt, bias, dy, Tout, stride, pl):
    from wav2letter_b200 import capi

    T, K = x.shape[1], wt.shape[2]
    try:
        capi.set_precision(prec)
        y = capi.conv_time_fwd(x, wt, bias, Tout, stride, pl)
        dx = capi.conv_time_dgrad(dy, wt, T, stride, pl)
        dwt, dbias = capi.conv_time_wgrad(x, dy, K, stride, pl)
    finally:
        capi.set_precision("tf32")
    return y, dx, dwt, dbias


@pytest.mark.parametrize("prec", ["f32", "tf32"])
@pytest.mark.parametrize("B,T,Cin,Cout,K,stride,W", [
    (2, 37, 10, 10, 21, 1, 80),    # T' not a multiple of any chunk
    (2, 1, 10, 14, 21, 1, 80),     # T' = 1
    (3, 2, 14, 18, 21, 2, 80),     # T' = 1, strided
    (2, 4000, 10, 10, 21, 1, 80),  # many chunks per weight-gradient CTA
    (1, 4000, 18, 18, 21, 1, 80),  # the same with two 16-channel M tiles
    (2, 601, 10, 14, 21, 2, 80),   # polyphase data gradient, odd T
    (2, 301, 14, 18, 21, 2, 80),
    (2, 301, 1, 10, 21, 2, 80),
    (2, 150, 18, 18, 21, 1, 8),
    (2, 300, 14, 14, 21, 1, 16),
    (2, 125, 27, 27, 11, 1, 80),
])
def test_conv_time_staging(B, T, Cin, Cout, K, stride, W, prec):
    g = torch.Generator(device="cuda").manual_seed(T * 31 + Cin * 7 + W)
    pl = (K - 1) // 2
    Tout = (T + 2 * pl - K) // stride + 1
    x = torch.randn((B, T, Cin, W), device="cuda", generator=g)
    wt = torch.randn((Cout, Cin, K), device="cuda", generator=g) * 0.1
    bias = torch.randn(Cout, device="cuda", generator=g)
    dy = torch.randn((B, Tout, Cout, W), device="cuda", generator=g)
    x64, w64, b64 = x.double().requires_grad_(True), wt.double().requires_grad_(True), bias.double().requires_grad_(True)
    pre = ref_conv(x64, w64, b64, stride, pl, Tout)
    pre.backward(dy.double())
    y, dx, dwt, dbias = run(prec, x, wt, bias, dy, Tout, stride, pl)
    tol = TOL[prec]
    assert rel(y, pre) < tol, rel(y, pre)
    assert rel(dx, x64.grad) < tol, rel(dx, x64.grad)
    assert rel(dwt, w64.grad) < tol, rel(dwt, w64.grad)
    assert rel(dbias, b64.grad) < tol


@pytest.mark.parametrize("prec", ["f32", "tf32"])
@pytest.mark.parametrize("T,Cin,Cout,stride", [(150, 10, 10, 1), (150, 18, 18, 1), (301, 10, 14, 2)])
def test_conv_time_windows_stay_inside_their_sample(T, Cin, Cout, stride, prec):
    """sample b is scaled by 1e3, 1e-3, 1e3, 1e-3: forward and data gradient are checked per sample (a frame of the
    neighbouring sample in a window would be a thousand-fold error there); the weight gradient sums over samples, so its
    dy is left unscaled and a large sample's frames leaking into a small one's window would be an O(1) error"""
    B, K, W = 4, 21, 80
    g = torch.Generator(device="cuda").manual_seed(T + Cin)
    pl = (K - 1) // 2
    Tout = (T + 2 * pl - K) // stride + 1
    scale = torch.tensor([1e3, 1e-3, 1e3, 1e-3], device="cuda")
    x = torch.randn((B, T, Cin, W), device="cuda", generator=g) * scale.view(B, 1, 1, 1)
    wt = torch.randn((Cout, Cin, K), device="cuda", generator=g) * 0.1
    bias = torch.zeros(Cout, device="cuda")
    dy1 = torch.randn((B, Tout, Cout, W), device="cuda", generator=g)
    dys = dy1 * scale.view(B, 1, 1, 1)
    x64, w64 = x.double().requires_grad_(True), wt.double().requires_grad_(True)
    pre = ref_conv(x64, w64, None, stride, pl, Tout)
    pre.backward(dy1.double())
    xs64 = x.double().requires_grad_(True)
    ref_conv(xs64, wt.double(), None, stride, pl, Tout).backward(dys.double())
    y, _, dwt, _ = run(prec, x, wt, bias, dy1, Tout, stride, pl)
    _, dx, _, _ = run(prec, x, wt, bias, dys, Tout, stride, pl)
    tol = TOL[prec]
    for b in range(B):
        assert rel(y[b], pre[b]) < tol, (b, rel(y[b], pre[b]))
        assert rel(dx[b], xs64.grad[b]) < tol, (b, rel(dx[b], xs64.grad[b]))
    assert rel(dwt, w64.grad) < tol, rel(dwt, w64.grad)
