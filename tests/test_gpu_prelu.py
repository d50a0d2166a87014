"""The `PR` opcode: the PReLU kernels against float64 torch, the fused dropout mask bit for bit against
dropout_reference.simt_scale, the a = 0 + dropout case a standalone Dropout would get wrong, run-to-run identical da, a
C2 -> PR -> DO 0 -> C2 net with slack rows against float64 torch, and the parser's refusal of `PR 2`."""
import numpy as np
import pytest
import torch

import dropout_reference as R
import oracle
from prelu_reference import ChannelNet, prelu

pytestmark = pytest.mark.gpu


def inputs(n, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(0, 1, n).astype(np.float32)
    x[rng.integers(0, n, n // 10)] = 0.0  # exact zeros: the x >= 0 branch
    g = rng.normal(0, 1, n).astype(np.float32)
    return torch.from_numpy(x).cuda(), torch.from_numpy(g).cuda()


@pytest.mark.parametrize("a", [0.25, 0.0, -0.3])
@pytest.mark.parametrize("n", [1, 7, 4099, 1 << 20])
def test_prelu_against_float64(a, n):
    from wav2letter_b200 import capi

    x, g = inputs(n, n)
    av = torch.tensor([a], dtype=torch.float32, device="cuda")
    y = capi.prelu_fwd(x, av)
    dx, da = capi.prelu_bwd(x, g, av)
    x64, g64 = x.double(), g.double()
    a = float(av)  # the float32 value of a
    assert torch.equal(y, prelu(x64, a).float())  # one rounding either way
    assert torch.equal(dx, torch.where(x64 >= 0, g64, a * g64).float())
    ref = float((torch.where(x64 < 0, x64, 0.0) * g64).sum())
    scale = float((x64.clamp_max(0).abs() * g64.abs()).sum())
    assert abs(float(da) - ref) <= 1e-6 * max(scale, 1.0)


@pytest.mark.parametrize("a", [0.25, 0.0])
def test_fused_dropout_mask_is_simt_scale(a):
    from wav2letter_b200 import capi

    n, p, seed = 100003, 0.3, 0x1234ABCD5678
    x, g = inputs(n, 3)
    av = torch.tensor([a], dtype=torch.float32, device="cuda")
    m = torch.from_numpy(R.simt_scale(seed, np.arange(n, dtype=np.uint64), p)).cuda()
    y = capi.prelu_fwd(x, av, p, seed)
    assert torch.equal(y, prelu(x, torch.tensor(a, device="cuda")) * m)
    dx, da = capi.prelu_bwd(x, g, av, p, seed)
    gm = g * m
    assert torch.equal(dx, torch.where(x >= 0, gm, a * gm))
    # a = 0: the output is exactly zero on every x <= 0 and on every dropped element, yet kept x = 0 elements pass their
    # gradient and every kept x < 0 contributes to da — what a mask read off the output ("zero = dropped") would lose
    ref = float((torch.where(x < 0, x, 0).double() * gm.double()).sum())
    assert abs(float(da) - ref) <= 1e-5 * float((x.double().abs() * gm.double().abs()).sum())
    if a == 0.0:
        kept_zero = (x == 0) & (m > 0)
        assert kept_zero.any() and torch.equal(dx[kept_zero], gm[kept_zero])
        assert float(da) != 0.0


def test_da_is_identical_run_to_run():
    from wav2letter_b200 import capi

    x, g = inputs(3_000_001, 9)
    av = torch.tensor([0.25], dtype=torch.float32, device="cuda")
    a = [capi.prelu_bwd(x, g, av, 0.5, 77) for _ in range(3)]
    assert all(torch.equal(a[0][0], b[0]) and torch.equal(a[0][1], b[1]) for b in a[1:])


ARCH = """V -1 1 NFEAT 0
C2 NFEAT 16 5 1 1 1 -1 0
PR
DO 0.0
C2 16 12 3 1 1 1 -1 0
PR 1 -0.1
RO 2 0 3 1
L 12 NLABEL
"""


def test_c2_prelu_c2_with_slack_rows_against_float64():
    """B > 1 with W = 1 convolutions: the batch carries slack rows, which the second convolution must not read as data"""
    from wav2letter_b200.trainer import Trainer

    F_, N, B, T = 16, 6, 3, 37  # (the channel-major head takes a multiple of 8 features)
    tr = Trainer(ARCH, F_, N, "ctc", "none", lr=0.0, maxgradnorm=0.0, precision="f32")
    assert "PReLU" in tr.describe()
    rng = np.random.default_rng(4)
    feat = torch.from_numpy(rng.standard_normal((B, 1, F_, T), dtype=np.float32)).cuda()
    y = torch.from_numpy(rng.integers(0, N - 1, (B, 5)).astype(np.int32)).cuda()
    flat, layout = tr.get_flat(0, 0).clone(), tr.layout(0)
    assert [n for _, n, _ in layout] == [16 * F_ * 5, 16, 1, 12 * 16 * 3, 12, 1, N * 12, N]
    assert float(flat[layout[2][0]]) == 0.25 and float(flat[layout[5][0]]) == pytest.approx(-0.1)
    emis = tr.forward(feat).clone()
    tr.step(feat, y, True, float(B))
    grads = tr.get_flat(0, 1).double()
    ref = ChannelNet(ARCH, F_, N, flat, layout)
    e64 = ref.forward(feat)
    assert e64.shape == emis.shape
    assert float((emis.double() - e64).abs().max()) <= 2e-4 * float(e64.abs().max())
    _, ode = oracle.ctc(e64.detach().float().cpu().numpy(), y.cpu().numpy(), "none")
    e64.backward(torch.from_numpy(ode).to(e64.device).double())
    g64 = ref.grads_flat(layout, flat.numel())
    gmax = float(g64.abs().max())
    assert float((grads - g64).abs().max()) <= 1e-3 * gmax
    for o, n, _ in layout:  # every parameter, the two PReLU scalars included
        err = float((grads[o:o + n] - g64[o:o + n]).norm())
        assert err <= 1e-3 * max(float(g64[o:o + n].norm()), 1e-3 * gmax), (o, n)
    tr.close()


def test_pr_with_two_parameters_is_refused():
    from wav2letter_b200.capi import W2LError
    from wav2letter_b200.trainer import Trainer

    with pytest.raises(W2LError) as ei:
        Trainer("V -1 1 NFEAT 0\nC2 NFEAT 4 5 1 1 1 -1 0\nPR 2\nRO 2 0 3 1\nL 4 NLABEL\n", 16, 6, "ctc")
    assert "PR with 2 parameters is not covered" in str(ei.value)


def test_streaming_export_refuses_pr(tmp_path):
    """PR is outside the streaming export's subset: the export and w2l_stream_create fail with an error, not a crash"""
    from wav2letter_b200.capi import W2LError
    from wav2letter_b200.streaming import StreamingAM
    from wav2letter_b200.trainer import Trainer

    tr = Trainer(ARCH, 16, 6, "ctc")
    with pytest.raises(W2LError):
        tr.export_streaming(str(tmp_path))
    with pytest.raises(W2LError):
        StreamingAM(tr, 2, 16)
    tr.close()
