"""CPU-side checks of the C ABI: the library loads, exports every symbol include/w2l_b200.h
declares, reports workspace sizes, and rejects bad arguments with the documented codes —
no kernel is launched, so they run without a GPU."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    txt = open(os.path.join(ROOT, "include", "w2l_b200.h")).read()
    return sorted(set(re.findall(r"W2L_API\s+[\w\s\*]+?\b(w2l_\w+)\s*\(", txt)))


def test_library_exports_every_declared_symbol():
    from wav2letter_b200 import capi

    syms = header_symbols()
    assert len(syms) >= 14
    for s in syms:
        assert hasattr(capi.lib, s), f"{s} declared in include/w2l_b200.h but not exported"
    assert sorted(capi.EXPORTS) == syms


def test_golden_fixture_matches_oracle():
    import oracle

    g = np.load(os.path.join(ROOT, "tests", "golden", "criterion_goldens.npz"))
    loss, de, dtr = oracle.asg(g["asg_emis"], g["asg_target"], g["asg_trans"], "target_sz_sqrt")
    np.testing.assert_array_equal(loss, g["asg_loss"])
    np.testing.assert_array_equal(de, g["asg_d_emis"])
    np.testing.assert_array_equal(oracle.fcc_viterbi(g["asg_emis"], g["asg_trans"]), g["asg_viterbi"])
    l2, d2 = oracle.ctc(g["ctc_emis"], g["ctc_target"], "target_sz")
    np.testing.assert_array_equal(l2, g["ctc_loss"])


def test_workspace_sizes_and_argument_errors():
    from wav2letter_b200 import capi

    lib = capi.lib
    assert lib.w2l_version() >= 100
    assert lib.w2l_asg_workspace_size(64, 1500, 30, 250) > 64 * 1500 * 32 * 4 * 4
    assert lib.w2l_asg_workspace_size(0, 10, 30, 5) == 0
    assert lib.w2l_ctc_workspace_size(8, 100, 31, 20) > 0
    assert lib.w2l_fcc_viterbi_workspace_size(2, 100, 30) >= 2 * 100 * 32
    # argument validation happens before any CUDA call
    vp = ctypes.c_void_p
    one = vp(256)  # never dereferenced: validation fails first
    rc = lib.w2l_asg_forward_backward(None, capi.TERM_ASG, 0, 10, 30, 5, 0, one, one, one, None, one, one, one, one, 1 << 30)
    assert rc == 1 and b"positive" in lib.w2l_last_error()
    rc = lib.w2l_asg_forward_backward(None, capi.TERM_ASG, 2, 10, 40, 5, 0, one, one, one, None, one, one, one, one, 1 << 30)
    assert rc == 4  # N > 32 unsupported
    rc = lib.w2l_asg_forward_backward(None, capi.TERM_ASG, 2, 10, 30, 5, 0, one, one, one, None, one, one, one, one, 16)
    assert rc == 2 and b"workspace" in lib.w2l_last_error()
    rc = lib.w2l_asg_forward_backward(None, capi.TERM_ASG, 2, 10, 30, 5, 0, one, None, one, None, one, one, one, one, 1 << 30)
    assert rc == 1  # FAC without target
    rc = lib.w2l_asg_forward_backward(None, 8, 2, 10, 30, 5, 0, one, one, one, None, one, one, one, one, 1 << 30)
    assert rc == 1
    rc = lib.w2l_ctc_forward_backward(None, 2, 10, 1, 5, 0, one, one, None, one, one, one, 1 << 30)
    assert rc == 1
    rc = lib.w2l_ctc_forward_backward(None, 2, 10, 31, 5, 9, one, one, None, one, one, one, 1 << 30)
    assert rc == 1
    rc = lib.w2l_fcc_viterbi(None, 1, 10, 33, one, one, one, one, 1 << 20)
    assert rc == 4


def test_capi_rejects_cpu_tensors():
    import torch

    from wav2letter_b200 import capi

    with pytest.raises(TypeError):
        capi.asg_forward_backward(torch.zeros(1, 2, 3), torch.zeros(1, 1, dtype=torch.int32), torch.zeros(3, 3))
