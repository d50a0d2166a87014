"""A trainer with 39 tokens (the folded TIMIT phone set) trains through the 64-wide ASG / LinSeg calls: its loss is
w2l_asg64_forward_backward's on its own emissions and transitions, it falls when trained, and the forced alignment
still equals w2l_fac_viterbi."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ARCH = """V -1 NFEAT 1 0
C2 1 8 5 1 2 1 -1 -1
R
DO 0.0
LN 3
V 0 320 1 0
RO 1 0 3 2
L 320 NLABEL
"""
N, F, B, T, L = 39, 40, 4, 120, 20


@pytest.mark.parametrize("criterion", ["asg", "linseg"])
def test_trainer_with_39_tokens(criterion):
    from wav2letter_b200 import capi
    from wav2letter_b200.trainer import Trainer

    rng = np.random.default_rng(5)
    feat = torch.from_numpy(rng.normal(0, 1, (B, 1, F, T)).astype(np.float32)).cuda()
    y = rng.integers(0, N, (B, L)).astype(np.int32)
    y[1, 12:] = -1
    dy = torch.from_numpy(y).cuda()
    tr = Trainer(ARCH, F, N, criterion, "target_sz_sqrt", transdiag=2.0, lr=0.1, lrcrit=0.1, momentum=0.5, maxgradnorm=1.0)
    first = tr.step(feat, dy, train=False).clone()
    emis = tr.forward(feat).contiguous()
    trans = tr.get_flat(which=1)[: N * N].view(N, N).contiguous()
    target = capi.linseg_target(dy, emis.shape[1]) if criterion == "linseg" else dy
    ref, _, _ = capi.asg64_forward_backward(emis, target, trans, "target_sz_sqrt", need_grad=False)
    torch.testing.assert_close(first, ref, rtol=1e-5, atol=1e-5)
    for _ in range(30):
        tr.step(feat, dy, train=True)
    last = tr.step(feat, dy, train=False)
    assert torch.isfinite(last).all() and last.sum().item() < first.sum().item()
    if criterion == "asg":
        emis = tr.forward(feat).contiguous()
        trans = tr.get_flat(which=1)[: N * N].view(N, N).contiguous()
        path, idx = tr.align(feat, dy)
        fp, fi = capi.fac_viterbi(emis, dy, trans, return_index=True)
        assert torch.equal(path, fp) and torch.equal(idx, fi)
    tr.close()
