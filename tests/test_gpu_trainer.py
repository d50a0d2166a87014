"""End-to-end parity of the C++ training step (arch parser -> TDS network -> CTC / ASG criterion -> backward ->
clip -> SGD) against a plain PyTorch float64 reference of the same network built from the same parameters.
Tolerances: emissions / loss 5e-3 relative, all gradients together 2e-2, any single parameter 0.25 (of its own scale).  The dense
contractions run in TF32 on the tensor cores (10-bit mantissa operands), and the back-propagated error through
LayerNorm's mean subtractions is what cuBLAS/cuDNN-TF32 shows too: scripts/diag_trainer.py prints this kernel's
per-parameter error next to torch's own fp32+TF32 error vs float64 on the same network — they agree to 2-3
digits."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle

pytestmark = pytest.mark.gpu

ARCH = """V -1 NFEAT 1 0
C2 1 4 5 1 2 1 -1 -1
R
DO 0.0
LN 3
TDS 4 5 80 0.0
C2 4 8 5 1 2 1 -1 -1
R
DO 0.0
LN 3
TDS 8 5 80 0.0
TDS 8 5 80 0.0
V 0 640 1 0
RO 1 0 3 2
L 640 NLABEL
"""


def rel(a, b):
    a, b = a.detach(), b.detach()
    return float((a.double() - b.double()).abs().max() / max(1e-6, float(b.double().abs().max())))


def same_pad(T, k, s):
    rem = T % s
    tot = (k - 1) - (s if rem == 0 else rem) + 1
    return max((tot + 1) // 2, 0)


def conv_ref(x, w, b, s):
    """x [B,T,C,W]; w [cout,cin,k]"""
    T, k = x.shape[1], w.shape[2]
    p = same_pad(T, k, s)
    xin = F.pad(x.permute(0, 2, 1, 3), (0, 0, p, p))
    return F.conv2d(xin, w.unsqueeze(-1), b, stride=(s, 1)).permute(0, 2, 1, 3)


def ln_ref(x, g, b):
    return F.layer_norm(x, x.shape[1:], eps=1e-5) * g + b


class TorchTDS:
    """float64 reference of ARCH; parameters taken from the trainer's flat arena in module order."""

    def __init__(self, flat, layout):
        self.p = []
        for off, n, dims in layout:
            self.p.append(flat[off:off + n].double().clone().requires_grad_(True))
        self.layout = layout

    def forward(self, feat):
        """feat [B,1,F,T] -> logits [B,T',N]"""
        it = iter(range(len(self.p)))
        P = lambda: self.p[next(it)]
        x = feat.double().permute(0, 3, 1, 2)  # [B,T,1,F]

        def conv(x, cin, cout, k, s):
            return conv_ref(x, P().view(cout, cin, k), P().view(cout), s)

        def tds(x, c, k):
            y1 = conv(x, c, c, k, 1).clamp_min(0)
            z = ln_ref(x + y1, P(), P())
            B, T = z.shape[:2]
            W1, b1, W2, b2 = P().view(c * 80, c * 80), P(), P().view(c * 80, c * 80), P()
            h = (z.reshape(B, T, -1) @ W1.t() + b1).clamp_min(0)
            u = h @ W2.t() + b2
            return ln_ref(z + u.view_as(z), P(), P())

        x = conv(x, 1, 4, 5, 2).clamp_min(0)
        x = ln_ref(x, P(), P())
        x = tds(x, 4, 5)
        x = conv(x, 4, 8, 5, 2).clamp_min(0)
        x = ln_ref(x, P(), P())
        x = tds(x, 8, 5)
        x = tds(x, 8, 5)
        B, T = x.shape[:2]
        W, b = P(), P()
        N = b.numel()
        return x.reshape(B, T, -1) @ W.view(N, 640).t() + b


# streaming TDS family (recipes/streaming_convnets/librispeech/am_500ms_future_context.arch): explicit PD padding
# before valid strided convolutions, per-frame LayerNorm (`LN 1 2`, TDS lNormIncludeTime = 0), limited right context
STREAMING_ARCH = """V -1 NFEAT 1 0
PD 0 5 3
C2 1 4 10 1 2 1 0 0
R
DO 0.0
LN 1 2
TDS 4 9 80 0.0 0 1 0
PD 0 7 1
C2 4 8 10 1 2 1 0 0
R
DO 0.0
LN 1 2
TDS 8 9 80 0.0 0 1 0
TDS 8 5 80 0.0 0 0 0
V 0 640 1 0
RO 1 0 3 2
L 640 NLABEL
"""


class TorchStreamingTDS(TorchTDS):
    def forward(self, feat):
        it = iter(range(len(self.p)))
        P = lambda: self.p[next(it)]
        x = feat.double().permute(0, 3, 1, 2)  # [B,T,1,F]

        def conv(x, cin, cout, k, s, pl, pr):
            xin = F.pad(x.permute(0, 2, 1, 3), (0, 0, pl, pr))
            return F.conv2d(xin, P().view(cout, cin, k).unsqueeze(-1), P().view(cout), stride=(s, 1)).permute(0, 2, 1, 3)

        def ln(x, g, b):  # per frame over (C, W)
            return F.layer_norm(x, x.shape[2:], eps=1e-5) * g + b

        def tds(x, c, k, rpad):
            y1 = conv(x, c, c, k, 1, k - 1 - rpad, rpad).clamp_min(0)
            z = ln(x + y1, P(), P())
            B, T = z.shape[:2]
            W1, b1, W2, b2 = P().view(c * 80, c * 80), P(), P().view(c * 80, c * 80), P()
            h = (z.reshape(B, T, -1) @ W1.t() + b1).clamp_min(0)
            u = h @ W2.t() + b2
            return ln(z + u.view_as(z), P(), P())

        x = conv(x, 1, 4, 10, 2, 5, 3).clamp_min(0)
        x = ln(x, P(), P())
        x = tds(x, 4, 9, 1)
        x = conv(x, 4, 8, 10, 2, 7, 1).clamp_min(0)
        x = ln(x, P(), P())
        x = tds(x, 8, 9, 1)
        x = tds(x, 8, 5, 0)
        B, T = x.shape[:2]
        W, b = P(), P()
        N = b.numel()
        return x.reshape(B, T, -1) @ W.view(N, 640).t() + b


def make_batch(B, T, N, L, seed, blank):
    g = torch.Generator(device="cuda").manual_seed(seed)
    feat = torch.randn((B, 1, 80, T), device="cuda", generator=g)
    hi = N - 1 if blank else N
    tgt = torch.randint(0, hi, (B, L), device="cuda", generator=g, dtype=torch.int32)
    tgt[1, L // 2:] = -1
    return feat, tgt


# precision "f32" (fp32-accurate contractions) pins the arithmetic: every parameter within 1e-2 of its own gradient scale
# (floor: 1e-3 of the net's largest gradient entry).  "tf32" is the same graph with 10-bit operand mantissas: its
# per-parameter deviation is rounding only (the exact path is pinned by "f32") and is bounded loosely.
PREC_TOL = {"f32": dict(emis=3e-4, per_param=5e-2, floor=1e-2, overall=1e-2), "tf32": dict(emis=5e-3, per_param=0.6, floor=1e-2, overall=3e-2)}


@pytest.mark.parametrize("precision", ["f32", "tf32"])
@pytest.mark.parametrize("criterion,N,arch_name", [("ctc", 12, "tds"), ("asg", 8, "tds"), ("ctc", 12, "streaming")])
def test_train_step_matches_torch_reference(criterion, N, arch_name, precision):
    from wav2letter_b200.trainer import Trainer

    B, T, L = 3, 64, 5
    tol = PREC_TOL[precision]
    arch_text, ref_cls = (ARCH, TorchTDS) if arch_name == "tds" else (STREAMING_ARCH, TorchStreamingTDS)
    tr = Trainer(arch_text, 80, N, criterion, "target_sz" if criterion == "ctc" else "none", transdiag=1.0, lr=0.0, lrcrit=0.0,
                 precision=precision)
    feat, tgt = make_batch(B, T, N, L, 1, criterion == "ctc")
    flat0 = tr.get_flat(0, 0).clone()
    loss = tr.step(feat, tgt, train=True)
    torch.cuda.synchronize()
    grads = tr.get_flat(0, 1)
    assert torch.equal(tr.get_flat(0, 0), flat0)  # lr = 0
    ref = ref_cls(flat0, tr.layout(0))
    logits = ref.forward(feat)
    e = logits.detach().float().cpu().numpy()
    y = tgt.cpu().numpy()
    if criterion == "ctc":
        ol, ode = oracle.ctc(e, y, "target_sz")
    else:
        trans = tr.get_flat(1, 0).view(N, N).cpu().numpy()
        ol, ode, odt = oracle.asg(e, y, trans, "none")
        assert rel(tr.get_flat(1, 1), torch.from_numpy(odt).flatten().cuda()) < 5e-3
    # emissions and loss
    got = tr.forward(feat)
    assert rel(got, logits) < tol["emis"], rel(got, logits)
    assert rel(loss, torch.from_numpy(ol).cuda()) < tol["emis"], (loss, ol)
    # gradients of every parameter: chain the oracle's d_emis through the float64 torch graph
    logits.backward(torch.from_numpy(ode).double().cuda())
    full = torch.cat([p.grad.flatten() for p in ref.p])
    mine = torch.cat([grads[off:off + n] for off, n, _ in tr.layout(0)])
    gscale = float(full.abs().max())
    for (off, n, dims), p in zip(tr.layout(0), ref.p):
        # scalar LayerNorm gains/biases are sums with heavy cancellation: measure against the larger of the
        # parameter's own gradient scale and 1% of the global one
        # relative L2 error per parameter (floored): max-abs is hypersensitive to single ReLU-kink sign flips at these tiny sizes
        denom = max(float(p.grad.norm()), tol["floor"] * gscale * n ** 0.5)
        gerr = float((grads[off:off + n].double() - p.grad.flatten()).norm()) / denom
        assert gerr < tol["per_param"], f"{precision}: param at {off} dims {dims}: grad rel err {gerr}"
    assert rel(mine, full) < tol["overall"], rel(mine, full)


def test_training_reduces_loss_and_dropout_runs():
    from wav2letter_b200.trainer import Trainer

    arch = ARCH.replace("DO 0.0", "DO 0.1").replace("80 0.0", "80 0.1")
    tr = Trainer(arch, 80, 12, "ctc", "none", lr=0.02, momentum=0.5, maxgradnorm=5.0)
    feat, tgt = make_batch(4, 96, 12, 6, 3, True)
    first = tr.step(feat, tgt, train=False).sum().item()
    for _ in range(40):
        tr.step(feat, tgt, train=True)
    last = tr.step(feat, tgt, train=False).sum().item()
    assert np.isfinite(last) and last < 0.7 * first, (first, last)


def test_arch_errors():
    from wav2letter_b200 import W2LError
    from wav2letter_b200.trainer import Trainer

    with pytest.raises(W2LError):
        Trainer("TR 4 4 8 2 100\n", 80, 12)  # transformer blocks are outside the hot-path subset
    with pytest.raises(W2LError):
        Trainer("V -1 NFEAT 1 0\nPD 0 3 1\nR\n", 80, 12)  # PD must be followed by the convolution it pads
    Trainer("V -1 NFEAT 1 0\nL 78 12\n", 78, 12).close()  # Linear rows that are not TMA rows go through padded copies
