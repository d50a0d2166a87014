"""CPU oracle — TEST INFRASTRUCTURE ONLY.

ctypes front-end for ``oracle/libw2l_oracle.so`` (built from ``oracle/w2l_oracle.c``; see that
file's header for the reference citations and the "parity unpinned" statement).

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this package.  The product package ``wav2letter_b200``
never does.
"""
from __future__ import annotations

import atexit
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libw2l_oracle.so")

SCALE_MODES = {"none": 0, "input_sz": 1, "input_sz_sqrt": 2, "target_sz": 3, "target_sz_sqrt": 4}
TERM_FCC, TERM_FAC = 1, 2

_lib = None


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "w2l_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s", "-B" if force else "-s"])
    return _SO


_native_dir = None


def build_native() -> str:
    """-march=native build for the host it is called on (bench.py's CPU legs; BASELINE.md §4), compiled into one
    temporary directory per process (removed at exit) so that a read-only source tree works"""
    global _native_dir
    if _native_dir is None:
        _native_dir = tempfile.mkdtemp(prefix="w2l_oracle_")
        atexit.register(shutil.rmtree, _native_dir, True)
    so = os.path.join(_native_dir, "libw2l_oracle_native.so")
    if not os.path.exists(so):
        subprocess.check_call(["make", "-C", _HERE, "-s", "-B", "native", f"NATIVE_SO={so}"])
    return so


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        so = _SO
        if os.environ.get("W2L_ORACLE_NATIVE") == "1":  # set by bench.py only
            try:
                so = build_native()
            except Exception:
                so = _SO
        if so == _SO:
            build()
        _lib = ctypes.CDLL(so)
        _lib.oracle_scale.restype = ctypes.c_double
        _lib.oracle_scale.argtypes = [ctypes.c_int] * 3
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def num_threads() -> int:
    return lib().oracle_num_threads()


def set_num_threads(n: int) -> None:
    lib().oracle_set_num_threads(int(n))


def target_sizes(target, T: int):
    target = _i32(target)
    B, L = target.shape
    out = np.zeros(B, np.int32)
    lib().oracle_target_sizes(B, L, int(T), _p(target), _p(out))
    return out


def ctc_target_sizes(target, T: int):
    target = _i32(target)
    B, L = target.shape
    out = np.zeros(B, np.int32)
    lib().oracle_ctc_target_sizes(B, L, int(T), _p(target), _p(out))
    return out


def _asg(terms, emis, target, trans, scale_mode, dloss, backward):
    emis = _f32(emis)
    trans = _f32(trans)
    B, T, N = emis.shape
    assert trans.shape == (N, N)
    if target is not None:
        target = _i32(target)
        assert target.shape[0] == B
        L = target.shape[1]
    else:
        L = 0
    if dloss is not None:
        dloss = _f32(dloss)
    loss = np.zeros(B, np.float32)
    d_emis = np.zeros_like(emis) if backward else None
    d_trans = np.zeros_like(trans) if backward else None
    mode = SCALE_MODES[scale_mode] if isinstance(scale_mode, str) else int(scale_mode)
    rc = lib().oracle_asg(terms, B, T, N, L, mode, _p(emis), _p(target), _p(trans), _p(dloss), _p(loss),
                          _p(d_emis), _p(d_trans))
    if rc != 0:
        raise ValueError("oracle_asg: invalid arguments")
    return (loss, d_emis, d_trans) if backward else loss


def asg(emis, target, trans, scale_mode="none", dloss=None, backward=True):
    """ASG = FCC - FAC. Returns (loss[B], d_emis[B,T,N], d_trans[N,N]) or loss only."""
    return _asg(TERM_FCC | TERM_FAC, emis, target, trans, scale_mode, dloss, backward)


def fcc(emis, trans, scale_mode="none", target=None, dloss=None, backward=True):
    return _asg(TERM_FCC, emis, target, trans, scale_mode, dloss, backward)


def fac(emis, target, trans, scale_mode="none", dloss=None, backward=True):
    return _asg(TERM_FAC, emis, target, trans, scale_mode, dloss, backward)


def fcc_viterbi(emis, trans):
    emis = _f32(emis)
    trans = _f32(trans)
    B, T, N = emis.shape
    path = np.zeros((B, T), np.int32)
    if lib().oracle_fcc_viterbi(B, T, N, _p(emis), _p(trans), _p(path)) != 0:
        raise ValueError("oracle_fcc_viterbi: invalid arguments")
    return path


def fac_viterbi(emis, target, trans, return_index=False):
    emis = _f32(emis)
    trans = _f32(trans)
    target = _i32(target)
    B, T, N = emis.shape
    L = target.shape[1]
    path = np.zeros((B, T), np.int32)
    idx = np.zeros((B, T), np.int32)
    if lib().oracle_fac_viterbi(B, T, N, L, _p(emis), _p(target), _p(trans), _p(path), _p(idx)) != 0:
        raise ValueError("oracle_fac_viterbi: invalid arguments")
    return (path, idx) if return_index else path


def ctc(emis, target, scale_mode="none", dloss=None, backward=True):
    """CTC on raw activations (internal log-softmax, blank = N-1)."""
    emis = _f32(emis)
    B, T, N = emis.shape
    if target is not None:
        target = _i32(target)
        L = target.shape[1]
    else:
        L = 0
    if dloss is not None:
        dloss = _f32(dloss)
    loss = np.zeros(B, np.float32)
    d_emis = np.zeros_like(emis) if backward else None
    mode = SCALE_MODES[scale_mode] if isinstance(scale_mode, str) else int(scale_mode)
    if lib().oracle_ctc(B, T, N, L, mode, _p(emis), _p(target), _p(dloss), _p(loss), _p(d_emis)) != 0:
        raise ValueError("oracle_ctc: invalid arguments")
    return (loss, d_emis) if backward else loss


def argmax_path(emis):
    emis = _f32(emis)
    B, T, N = emis.shape
    path = np.zeros((B, T), np.int32)
    lib().oracle_argmax_path(B, T, N, _p(emis), _p(path))
    return path


def linseg_target(target, T: int):
    target = _i32(target)
    B, L = target.shape
    out = np.zeros((B, int(T)), np.int32)
    lib().oracle_linseg_target(B, int(T), L, _p(target), _p(out))
    return out
