"""Conv1D + GLU acoustic-model family (recipes/conv_glu/{wsj,librispeech}/network.arch): WeightNorm-wrapped large-channel
time convolutions run as wgmma GEMMs on zero-copy im2col views, GLU (+dropout), Reorder, WeightNorm Linear head.
Kernel-level parity against float64 torch, then one whole train step (ASG criterion, 6 letter classes) against a float64
torch graph built from the same parameters.  Tolerances are the TF32 ones of test_gpu_trainer.py."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle

pytestmark = pytest.mark.gpu


def rel(a, b):
    a, b = a.detach(), b.detach()
    return float((a.double() - b.double()).abs().max() / max(1e-6, float(b.double().abs().max())))


def test_weightnorm_and_glu_kernels():
    from wav2letter_b200 import capi
    import ctypes

    g = torch.Generator(device="cuda").manual_seed(3)
    rows, ln = 37, 530
    v = torch.randn(rows, ln, device="cuda", generator=g)
    gg = torch.rand(rows, device="cuda", generator=g) + 0.5
    w = torch.empty_like(v)
    inv = torch.empty(rows, device="cuda")
    capi._check(capi.lib.w2l_weightnorm_fwd(capi._stream(), rows, ln, capi._ptr(v), capi._ptr(gg), capi._ptr(w), capi._ptr(inv)))
    v64, g64 = v.double().requires_grad_(True), gg.double().requires_grad_(True)
    wr = g64[:, None] * v64 / v64.norm(dim=1, keepdim=True)
    assert rel(w, wr) < 1e-5
    dw = torch.randn(rows, ln, device="cuda", generator=g)
    wr.backward(dw.double())
    dv, dg = torch.zeros_like(v), torch.zeros_like(gg)
    capi._check(capi.lib.w2l_weightnorm_bwd(capi._stream(), rows, ln, capi._ptr(v), capi._ptr(gg), capi._ptr(inv), capi._ptr(dw), capi._ptr(dv),
                                            capi._ptr(dg)))
    assert rel(dv, v64.grad) < 1e-4 and rel(dg, g64.grad) < 1e-4
    # GLU
    R, H = 501, 122
    x = torch.randn(R, 2 * H, device="cuda", generator=g)
    y = torch.empty(R, H, device="cuda")
    capi._check(capi.lib.w2l_glu_fwd(capi._stream(), R, H, capi._ptr(x), capi._ptr(y), 0.0, 0))
    x64 = x.double().requires_grad_(True)
    yr = F.glu(x64, dim=1)
    assert rel(y, yr) < 1e-5
    dy = torch.randn(R, H, device="cuda", generator=g)
    yr.backward(dy.double())
    dx = torch.empty_like(x)
    capi._check(capi.lib.w2l_glu_bwd(capi._stream(), R, H, capi._ptr(x), capi._ptr(dy), capi._ptr(dx), 0.0, 0))
    assert rel(dx, x64.grad) < 1e-5
    # dropout: forward and backward use the same mask, kept elements scaled by 1/(1-p)
    capi._check(capi.lib.w2l_glu_fwd(capi._stream(), R, H, capi._ptr(x), capi._ptr(y), 0.5, 11))
    capi._check(capi.lib.w2l_glu_bwd(capi._stream(), R, H, capi._ptr(x), capi._ptr(dy), capi._ptr(dx), 0.5, 11))
    kept = y != 0
    assert abs(float(kept.float().mean()) - 0.5) < 0.02
    assert rel(y[kept], 2 * yr[kept]) < 1e-5
    assert rel(dx[:, :H][kept], 2 * x64.grad[:, :H][kept]) < 1e-5 and float(dx[:, :H][~kept].abs().max()) == 0.0


ARCH = """V -1 1 NFEAT 0
WN 3 C NFEAT 24 5 1 -1
GLU 2
DO 0.0
WN 3 C 12 28 3 1 -1
GLU 2
DO 0.0
WN 3 C 14 40 4 1 0
GLU 2
DO 0.0
RO 2 0 3 1
WN 0 L 20 16
GLU 0
DO 0.0
WN 0 L 8 NLABEL
"""


class TorchConvGlu:
    """float64 reference of ARCH; parameters from the trainer's flat arena in module order (v, g, bias per layer)."""

    def __init__(self, flat, layout):
        self.p = [flat[off:off + n].double().clone().requires_grad_(True) for off, n, _ in layout]

    def forward(self, feat):
        it = iter(range(len(self.p)))
        P = lambda: self.p[next(it)]
        x = feat.double()[:, 0]  # [B, F, T]: features are channels

        def wn_conv(x, cin, cout, k, pad):
            v, g, b = P().view(cout, cin, k), P(), P()
            w = g.view(-1, 1, 1) * v / v.reshape(cout, -1).norm(dim=1).view(-1, 1, 1)
            return F.conv1d(F.pad(x, (pad, pad)), w, b)

        def wn_lin(x, nin, nout):
            v, g, b = P().view(nout, nin), P(), P()
            w = g.view(-1, 1) * v / v.norm(dim=1, keepdim=True)
            return x @ w.t() + b

        x = F.glu(wn_conv(x, 40, 24, 5, 2), dim=1)
        x = F.glu(wn_conv(x, 12, 28, 3, 1), dim=1)
        x = F.glu(wn_conv(x, 14, 40, 4, 0), dim=1)
        x = x.permute(0, 2, 1)  # [B, T', C]
        x = F.glu(wn_lin(x, 20, 16), dim=2)
        return wn_lin(x, 8, self.p[-1].numel())


PREC_TOL = {"f32": dict(emis=3e-4, per_param=5e-3, floor=1e-3, overall=1e-3), "tf32": dict(emis=5e-3, per_param=0.05, floor=1e-2, overall=2e-2),
            "bf16": dict(emis=3e-2, per_param=0.3, floor=1e-2, overall=1e-1)}


@pytest.mark.parametrize("precision", ["f32", "tf32", "bf16"])
def test_conv_glu_train_step_matches_torch_reference(precision):
    from wav2letter_b200.trainer import Trainer

    B, T, L, N = 3, 50, 5, 6
    tol = PREC_TOL[precision]
    tr = Trainer(ARCH, 40, N, "asg", "target_sz_sqrt", transdiag=1.0, lr=0.0, lrcrit=0.0, precision=precision)
    g = torch.Generator(device="cuda").manual_seed(2)
    feat = torch.randn((B, 1, 40, T), device="cuda", generator=g)
    tgt = torch.randint(0, N, (B, L), device="cuda", generator=g, dtype=torch.int32)
    tgt[1, 3:] = -1
    flat0 = tr.get_flat(0, 0).clone()
    loss = tr.step(feat, tgt, train=True)
    torch.cuda.synchronize()
    grads = tr.get_flat(0, 1)
    ref = TorchConvGlu(flat0, tr.layout(0))
    logits = ref.forward(feat)
    assert logits.shape == (B, T - 3, N)
    got = tr.forward(feat)
    assert rel(got, logits) < tol["emis"], rel(got, logits)
    trans = tr.get_flat(1, 0).view(N, N).cpu().numpy()
    ol, ode, odt = oracle.asg(logits.detach().float().cpu().numpy(), tgt.cpu().numpy(), trans, "target_sz_sqrt")
    assert rel(loss, torch.from_numpy(ol).cuda()) < tol["emis"]
    logits.backward(torch.from_numpy(ode).double().cuda())
    full = torch.cat([p.grad.flatten() for p in ref.p])
    mine = torch.cat([grads[off:off + n] for off, n, _ in tr.layout(0)])
    gscale = float(full.abs().max())
    for (off, n, dims), p in zip(tr.layout(0), ref.p):
        denom = max(float(p.grad.norm()), tol["floor"] * gscale * n ** 0.5)
        gerr = float((grads[off:off + n].double() - p.grad.flatten()).norm()) / denom
        assert gerr < tol["per_param"], f"{precision}: param at {off} dims {dims}: grad rel err {gerr}"
    assert rel(mine, full) < tol["overall"], rel(mine, full)


def test_conv_glu_training_reduces_loss_with_dropout():
    from wav2letter_b200.trainer import Trainer

    arch = ARCH.replace("DO 0.0", "DO 0.1")
    tr = Trainer(arch, 40, 6, "asg", "target_sz_sqrt", transdiag=1.0, lr=0.05, lrcrit=0.005, momentum=0.5, maxgradnorm=1.0)
    g = torch.Generator(device="cuda").manual_seed(4)
    feat = torch.randn((4, 1, 40, 60), device="cuda", generator=g)
    tgt = torch.randint(0, 6, (4, 6), device="cuda", generator=g, dtype=torch.int32)
    first = tr.step(feat, tgt, train=False).sum().item()
    for _ in range(40):
        tr.step(feat, tgt, train=True)
    last = tr.step(feat, tgt, train=False).sum().item()
    assert np.isfinite(last) and last < 0.7 * first, (first, last)
