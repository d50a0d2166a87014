"""CPU checks of the fp16 precision, the learning-rate schedule and the checkpoint versions: every new entry point rejects
bad arguments with W2L_ERR_INVALID_ARGUMENT before it touches the trainer or launches anything, so these run without a
GPU (the trainer handle below is never dereferenced)."""
import ctypes
import struct

import pytest

INVALID = 1
INT64_MAX = (1 << 63) - 1


def test_fp16_precision_and_kind_are_accepted_and_validated():
    from wav2letter_b200 import capi

    lib = capi.lib
    assert capi.PRECISIONS["fp16"] == 3 and capi.GEMM_KINDS["fp16"] == 4
    saved = lib.w2l_get_precision()
    try:
        assert lib.w2l_set_precision(3) == 0 and lib.w2l_get_precision() == 3
        assert lib.w2l_set_precision(4) == INVALID
    finally:
        lib.w2l_set_precision(saved)
    fake = ctypes.c_void_p(256)
    assert lib.w2l_trainer_set_precision(fake, 4) == INVALID
    # fp16 rows are TMA rows of 8 elements: ld = 12 passes for fp32 kinds, not for the 16-bit ones
    one = ctypes.c_void_p(256)
    rc = lib.w2l_gemm(None, 4, 0, 0, 64, 64, 64, one, 12, one, 64, one, 64, 0, None, 0, 0, None, 0, 0, 0, ctypes.c_float(1.0),
                      ctypes.c_float(0.0), ctypes.c_ulonglong(0), 0)
    assert rc == INVALID and b"16-byte" in lib.w2l_last_error()
    rc = lib.w2l_gemm(None, 5, 0, 0, 64, 64, 64, one, 64, one, 64, one, 64, 0, None, 0, 0, None, 0, 0, 0, ctypes.c_float(1.0),
                      ctypes.c_float(0.0), ctypes.c_ulonglong(0), 0)
    assert rc == INVALID and b"kind" in lib.w2l_last_error()
    assert lib.w2l_cast_fp16(None, 10, None, one) == INVALID
    assert lib.w2l_cast_fp16_rows(None, 4, 10, 10, 8, one, one) == INVALID  # padded row shorter than the row
    # the conv arrangement writes fp32 (0), bf16 (1) or fp16 (2) operands
    rc = lib.w2l_conv1d_arrange_ex(None, 8, 8, 3, 8, 8, 0, one, None, one, None, None, 3)
    assert rc == INVALID


@pytest.mark.parametrize("args", [
    (-1, 1.0, 10, 0, 10, 0, 1),          # warmup < 0
    (1, 0.0, 10, 0, 10, 0, 1),           # gamma <= 0
    (1, float("nan"), 10, 0, 10, 0, 1),  # gamma not finite
    (1, float("inf"), 10, 0, 10, 0, 1),
    (1, 0.5, 0, 0, 10, 0, 1),            # stepsize <= 0
    (1, 0.5, 10, 2, 10, 0, 1),           # lrcosine not 0 / 1
    (1, 0.5, 10, 1, 0, 0, 1),            # nbatches <= 0
    (1, 0.5, 10, 0, 10, -1, 1),          # lr_decay < 0
    (1, 0.5, 10, 0, 10, 0, 0),           # lr_decay_step <= 0
])
def test_set_schedule_rejects_bad_arguments(args):
    from wav2letter_b200 import capi

    assert capi.lib.w2l_trainer_set_schedule(ctypes.c_void_p(256), *args) == INVALID


def test_position_and_lr_entry_points_reject_bad_arguments():
    from wav2letter_b200 import capi

    lib, fake = capi.lib, ctypes.c_void_p(256)
    assert lib.w2l_trainer_set_schedule(None, 1, 1.0, INT64_MAX, 0, INT64_MAX, INT64_MAX, INT64_MAX) == INVALID
    assert lib.w2l_trainer_set_position(fake, -1, 0) == INVALID
    assert lib.w2l_trainer_set_position(fake, 0, -1) == INVALID
    assert lib.w2l_trainer_set_position(None, 0, 0) == INVALID
    assert lib.w2l_trainer_set_lr(fake, float("nan"), 0.1) == INVALID
    assert lib.w2l_trainer_set_lr(fake, 0.1, float("inf")) == INVALID
    assert lib.w2l_trainer_set_lr(None, 0.1, 0.1) == INVALID
    assert lib.w2l_trainer_lr(None, None, None) == INVALID
    assert lib.w2l_trainer_position(None, None, None) == INVALID


def _header(version, tail=b""):
    return b"W2LB200\0" + struct.pack("<I", version) + tail


@pytest.mark.parametrize("version", [0, 3])
def test_load_rejects_unknown_checkpoint_versions(tmp_path, version):
    from wav2letter_b200 import capi

    p = tmp_path / "ck.bin"
    p.write_bytes(_header(version, b"\0" * 64))
    assert not capi.lib.w2l_trainer_load(None, str(p).encode())
    assert b"unsupported version" in capi.lib.w2l_last_error()
    p.write_bytes(_header(2)[:-2])  # truncated inside the version
    assert not capi.lib.w2l_trainer_load(None, str(p).encode())


@pytest.mark.parametrize("args", [
    (2, 4096.0, 2000, 32000.0, 1e-4),           # on not 0 / 1
    (1, 0.0, 2000, 32000.0, 1e-4),              # initial scale <= 0
    (1, float("inf"), 2000, 32000.0, 1e-4),     # initial scale not finite
    (1, 4096.0, 0, 32000.0, 1e-4),              # update interval <= 0
    (1, 4096.0, 2000, 0.0, 1e-4),               # max scale <= 0
    (1, 4096.0, 2000, float("nan"), 1e-4),
    (1, 4096.0, 2000, 32000.0, -1.0),           # min scale < 0
    (1, 4096.0, 2000, 32000.0, float("nan")),
])
def test_set_amp_rejects_bad_arguments(args):
    from wav2letter_b200 import capi

    assert capi.lib.w2l_trainer_set_amp(ctypes.c_void_p(256), *args) == INVALID
    assert capi.lib.w2l_trainer_set_amp(None, 1, 4096.0, 2000, 32000.0, 1e-4) == INVALID
    assert capi.lib.w2l_trainer_amp_state(None, None, None, None, None) == INVALID
