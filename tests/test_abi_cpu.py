"""CPU-side checks of the C ABI: the library loads, binds every prototype include/w2l_b200.h
declares with the types it states, reports workspace sizes, and rejects bad arguments with the documented codes —
no kernel is launched, so they run without a GPU."""
import ctypes
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_binds_every_declared_prototype():
    from wav2letter_b200 import capi

    txt = open(os.path.join(ROOT, "include", "w2l_b200.h")).read()
    assert len(capi.PROTOTYPES) >= 14
    assert len(capi.PROTOTYPES) == txt.count("W2L_API ") - txt.count("#define W2L_API ")  # the reader saw every declaration
    for s, (restype, argtypes) in capi.PROTOTYPES.items():
        assert hasattr(capi.lib, s), f"{s} declared in include/w2l_b200.h but not exported"
        fn = getattr(capi.lib, s)
        assert fn.restype is restype and tuple(fn.argtypes) == argtypes, s


def test_prototype_types():
    """literal signatures, so that a reader that maps every function the same wrong way cannot pass"""
    from ctypes import c_char_p, c_double, c_float, c_int, c_longlong, c_size_t, c_ulonglong, c_void_p

    from wav2letter_b200 import capi

    P = capi.PROTOTYPES
    vp, i = c_void_p, c_int
    assert P["w2l_gemm"] == (c_int, (vp, i, i, i, i, i, i, vp, i, vp, i, vp, i, i, vp, i, i, vp, i, i, i,
                                     c_float, c_float, c_ulonglong, c_int))
    assert P["w2l_fill"] == (c_int, (c_void_p, c_longlong, c_float, c_void_p))
    assert P["w2l_set_seed"][1] == (c_ulonglong,)
    assert P["w2l_ema_update"][1][-1] is c_double
    assert P["w2l_trainer_create"][1][1] is c_char_p  # const char* arch_text
    for name, restype in (("w2l_last_error", c_char_p), ("w2l_trainer_describe", c_char_p), ("w2l_launch_count", c_longlong),
                          ("w2l_stream_state_bytes", c_longlong), ("w2l_asg_workspace_size", c_size_t),
                          ("w2l_trainer_create", c_void_p), ("w2l_trainer_destroy", None)):
        assert P[name][0] is restype, name


@pytest.mark.parametrize("decl", ["W2L_API int w2l_x(int32_t n);", "W2L_API int* w2l_x(void);", "W2L_API int w2l_x(int);",
                                  "W2L_API int w2l_x(float v[]);", "W2L_API int w2l_x(int (*cb)(int));"])
def test_header_reader_refuses_what_it_cannot_bind(decl):
    """a type outside the table, or a declaration the reader cannot parse, stops the import instead of going unbound"""
    from wav2letter_b200 import capi

    with pytest.raises(ImportError, match="w2l_x"):
        capi._read_header("/* a */\n" + decl + "\nW2L_API int w2l_ok(void);")


def test_header_constants():
    from wav2letter_b200 import capi

    assert (capi.W2L_OK, capi.W2L_ERR_UNSUPPORTED, capi.W2L_TERM_ASG, capi.W2L_SCALE_TARGET_SZ_SQRT, capi.W2L_GEMM_F32X3_SPLIT_B,
            capi.W2L_PRECISION_FP16, capi.W2L_LN_MAX_PARTS) == (0, 4, 3, 4, 3, 3, 80)
    assert capi.PRECISIONS == {"tf32": 0, "f32": 1, "fp32": 1, "bf16": 2, "fp16": 3}
    assert capi.GEMM_KINDS == {"tf32": 0, "f32x3": 1, "bf16": 2, "f32x3_split_b": 3, "fp16": 4}
    assert capi.SCALE_MODES == {"none": 0, "input_sz": 1, "input_sz_sqrt": 2, "target_sz": 3, "target_sz_sqrt": 4}
    assert (capi.TERM_FCC, capi.TERM_FAC, capi.TERM_ASG) == (1, 2, 3)


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
