"""The trainer in fp16 precision (W2L_PRECISION_FP16: the GEMM operands of every dense layer in fp16, fp32 accumulation;
everything else as in bf16 mode) on the four BASELINE archs, end to end against the float64 torch graph of
oracle/am_ref.py: emissions, loss and every parameter gradient (the harness of test_gpu_archs.py, run_case).

fp16 keeps 11 significand bits to bf16's 8, so its tolerances are tf32's (also 11 bits), and on the same inputs and
parameters its emission error must be below bf16's.  Repeating a step from the same parameters gives the same bits."""
import numpy as np
import pytest
import torch

import test_gpu_archs as archs_parity
from oracle import am_ref

pytestmark = pytest.mark.gpu

TOL = dict(emis=2e-2, loss=2e-2, overall=4e-2)


@pytest.mark.parametrize("name", sorted(archs_parity.CASES))
def test_arch_file_parity_fp16(name):
    rec = archs_parity.run_case(name, "fp16")
    assert np.isfinite(rec["loss"]).all()
    assert rec["emis_err"] <= TOL["emis"], rec
    assert rec["loss_err"] <= TOL["loss"], rec
    assert rec["grad_overall"] <= TOL["overall"], rec
    bf16 = archs_parity.run_case(name, "bf16")
    assert rec["emis_err"] < bf16["emis_err"], (rec["emis_err"], bf16["emis_err"])


@pytest.mark.parametrize("name", ["conv_glu_wsj", "streaming_tds_ctc"])
def test_fp16_steps_repeat_bit_for_bit(name):
    from wav2letter_b200 import archs
    from wav2letter_b200.trainer import Trainer

    gen, crit, _, _ = archs.BASELINE_ARCHS[name]
    F, N, B, T, L, mode, transdiag = archs_parity.CASES[name]
    # dropout and SpecAugment draw new masks at every step: off, so the two runs see the same network
    tr = Trainer(am_ref.zero_dropout(gen()), F, N, crit, mode, transdiag=transdiag, lr=0.1, lrcrit=0.01, maxgradnorm=1.0, precision="fp16")
    g = torch.Generator(device="cuda").manual_seed(5)
    feat = torch.randn((B, 1, F, T), device="cuda", generator=g)
    tgt = torch.randint(0, N - 1, (B, L), device="cuda", generator=g, dtype=torch.int32)
    flat0, crit0 = tr.get_flat(0, 0).clone(), tr.get_flat(1, 0).clone()
    runs = []
    for _ in range(2):
        tr.set_flat(flat0, 0)
        if crit0.numel():
            tr.set_flat(crit0, 1)
        emis = tr.forward(feat).clone()
        loss = tr.step(feat, tgt, True, float(B)).clone()
        runs.append((emis, loss, tr.get_flat(0, 1).clone(), tr.get_flat(0, 0).clone()))
    torch.cuda.synchronize()
    assert tr.skipped_steps() == 0
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    tr.close()
