"""wav2letter_b200 — H100-native (sm_90a) implementation of wav2letter's training hot path.

The product is ``libw2l_b200.so`` (hand-written CUDA behind the C ABI in ``include/w2l_b200.h``)
plus the C++ ``fl_compat`` layer that mirrors the reference's operator surface.  This Python
package is only the harness side: it loads the library with ctypes and passes torch device
pointers / streams to it (torch = device memory + streams + torch.distributed plumbing).
There is NO CPU or PyTorch fallback: if the library is missing, importing ``capi`` raises.
"""
from . import capi  # noqa: F401
from .capi import (  # noqa: F401
    SCALE_MODES,
    TERM_ASG,
    TERM_FAC,
    TERM_FCC,
    W2LError,
    argmax_path,
    asg_forward_backward,
    ctc_forward_backward,
    fac_viterbi,
    fcc_viterbi,
    launch_count,
    linseg_target,
    reset_launch_count,
)
