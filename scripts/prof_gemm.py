"""A few launches of the wgmma GEMM on the stage-1 FC shapes of the seq2seq_tds step, for `ncu --set full -k regex:gemm_wgmma`."""
import sys

import torch

sys.path.insert(0, ".")
import wav2letter_b200 as w  # noqa: E402

kind = sys.argv[1] if len(sys.argv) > 1 else "tf32"
dt = torch.bfloat16 if kind == "bf16" else torch.float32
for (M, N, K, a_mn, b_mn) in [(9600, 800, 800, False, False), (9600, 800, 800, False, True), (800, 800, 9600, True, True)]:
    A = torch.randn((K, M) if a_mn else (M, K), device="cuda").to(dt)
    B = torch.randn((K, N) if b_mn else (N, K), device="cuda").to(dt)
    for _ in range(2):
        w.capi.gemm(A, B, kind, a_mn, b_mn)
torch.cuda.synchronize()
