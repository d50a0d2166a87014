"""A few launches of the TDS time convolution (forward / stride-1 data gradient: wgmma kernel) at the stage shapes of the
seq2seq_tds step, for `ncu --set full -k regex:conv_wgmma_fwd`."""
import sys

import torch

sys.path.insert(0, ".")
from wav2letter_b200 import capi  # noqa: E402

capi._check(capi.lib.w2l_conv_set_path(3))
for (B, T, C, K) in [(16, 600, 10, 21), (16, 300, 14, 21), (16, 150, 18, 21)]:
    x = torch.randn(B, T, C, 80, device="cuda")
    wt = torch.randn(C, C, K, device="cuda") * 0.1
    bias = torch.randn(C, device="cuda")
    for _ in range(2):
        y = capi.conv_time_fwd(x, wt, bias, T, 1, 10, act=1, dropout_p=0.2, seed=5)
torch.cuda.synchronize()
