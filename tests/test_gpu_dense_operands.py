"""Linear layers whose rows are not TMA rows (4 floats, 8 bf16) go through zero-padded GEMM operands
(host/dense_operands.h).  They must compute what the same layers computed on aligned rows, bit for bit: the padded
route runs the same tiles with the same k order, and only the zero columns differ.

Arch A has 78 features and `L 78 78` / `L 78 30`: padded K in the forward of both Linear layers, a padded data
gradient for the second, padded weight gradients for both, and the 30-wide output gradient padded to 32 as a row
operand.  Arch B is the same network at 80 features (`L 80 80` / `L 80 30`): its parameters are A's with zero rows
and columns added, and it is fed A's features plus two zero feature columns.  The second View turns each frame's
features into channels ([1, F, T, B]), so the Linear layers see T frames of B samples.  The first Linear has no bias:
a bias gradient is a column sum whose kernel, and so its summation order, follows the width (78 or 80).
Each precision runs in a child process: the trainers draw their initial weights and dropout seeds from a per-process
counter, and the tests after this one must see the draws they see without it."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ARCH = "V -1 NFEAT 1 0\nV 0 1 {f} 0\nL {f} {f} 0\nL {f} 30\n"
N = 30


def padded_flat(flat_a, layout_a, layout_b):
    """B's parameters: A's, zero-padded (Linear weights are stored [nout][nin])"""
    out = torch.zeros(layout_b[-1][0] + layout_b[-1][1], device=flat_a.device)
    for (oa, na, da), (ob, nb, db) in zip(layout_a, layout_b):
        src = flat_a[oa:oa + na]
        if da[1] > 1:  # weight: dims [nin, nout]
            dst = out[ob:ob + nb].view(db[1], db[0])
            dst[:da[1], :da[0]] = src.view(da[1], da[0])
        else:
            out[ob:ob + na] = src
    return out


@pytest.mark.parametrize("precision", ["f32", "tf32", "bf16"])
def test_padded_linear_operands_match_aligned_bitwise(precision):
    r = subprocess.run([sys.executable, "-s", __file__, precision], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr


def compare(precision):
    from wav2letter_b200.trainer import Trainer

    B, T, L = 4, 256, 6  # 1024 rows: the weight gradients split K
    g = torch.Generator(device="cuda").manual_seed(7)
    feat_a = torch.randn((B, 1, 78, T), device="cuda", generator=g)
    feat_b = torch.zeros((B, 1, 80, T), device="cuda")
    feat_b[:, :, :78] = feat_a
    tgt = torch.randint(0, N - 1, (B, L), device="cuda", generator=g, dtype=torch.int32)
    tgt[1, L // 2:] = -1

    tr_a = Trainer(ARCH.format(f=78), 78, N, "ctc", "target_sz", lr=0.5, precision=precision)
    tr_b = Trainer(ARCH.format(f=80), 80, N, "ctc", "target_sz", lr=0.5, precision=precision)
    la, lb = tr_a.layout(0), tr_b.layout(0)
    tr_b.set_flat(padded_flat(tr_a.get_flat(0, 0), la, lb))

    assert torch.equal(tr_a.forward(feat_a), tr_b.forward(feat_b))
    loss_a = tr_a.step(feat_a, tgt).clone()
    loss_b = tr_b.step(feat_b, tgt).clone()
    torch.cuda.synchronize()
    assert torch.equal(loss_a, loss_b)

    for what in (1, 0):  # gradients, then the parameters after the step
        fa, fb = tr_a.get_flat(0, what), tr_b.get_flat(0, what)
        expect = padded_flat(fa, la, lb)
        for (ob, nb, db) in lb:
            assert torch.equal(fb[ob:ob + nb], expect[ob:ob + nb]), (what, db)
    assert torch.equal(tr_a.forward(feat_a), tr_b.forward(feat_b))
    tr_a.close()
    tr_b.close()


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    compare(sys.argv[1])
