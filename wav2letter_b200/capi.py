"""ctypes binding of include/w2l_b200.h for the Python harness (tests, bench, smoke).

The header is the one statement of the C ABI: at import, every `W2L_API` prototype in it sets the
restype / argtypes of its function in `lib` (PROTOTYPES), and its integer constants (enum entries,
`#define NAME <integer>`) become attributes of this module (W2L_OK, W2L_GEMM_FP16, W2L_LN_MAX_PARTS, ...).

Every function takes CUDA torch tensors, checks dtype/contiguity, and passes raw device
pointers and the current CUDA stream to the C ABI.  Workspaces are torch byte tensors owned
by the caller side (cached per size here), exactly as the C ABI demands.
"""
from __future__ import annotations

import ctypes
import os
import re

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libw2l_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "w2l_b200.h")

# C type -> ctypes type.  Parameters: `const char*` is a string, every other pointer a c_void_p.
_SCALARS = {"int": ctypes.c_int, "size_t": ctypes.c_size_t, "long long": ctypes.c_longlong,
            "unsigned long long": ctypes.c_ulonglong, "float": ctypes.c_float, "double": ctypes.c_double}
_RETURNS = dict(_SCALARS, **{"void": None, "void*": ctypes.c_void_p, "const char*": ctypes.c_char_p})


def _param(ctype: str):
    return ctypes.c_char_p if ctype == "const char*" else ctypes.c_void_p if ctype.endswith("*") else _SCALARS[ctype]


def _read_header(text: str):
    """({name: (restype, argtypes)} of every W2L_API declaration, {name: value} of every integer constant).
    A declaration that is not `ret name(type name, ...);` over the mapped types raises ImportError, so none goes unbound."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    prototypes = {}
    for decl in re.findall(r"(?<!#define )\bW2L_API\b[^;]*;", text):
        decl = " ".join(decl.replace("*", "* ").split()).replace(" *", "*")  # single spaces, pointers written `T*`
        m = re.fullmatch(r"W2L_API (.+) (w2l_\w+) ?\((.*)\);", decl)
        try:
            params = [] if m.group(3) == "void" else [re.fullmatch(r"(.+) \w+", p.strip()).group(1) for p in m.group(3).split(",")]
            prototypes[m.group(2)] = (_RETURNS[m.group(1)], tuple(map(_param, params)))
        except (AttributeError, KeyError):  # a regex did not match, or a type outside _SCALARS / _RETURNS
            raise ImportError(f"{HEADER_PATH}: cannot bind `{decl}`: not a prototype over the types capi.py maps") from None
    constants = {}
    for body in re.findall(r"\benum\s*\{([^}]*)\}", text):
        for entry in filter(str.strip, body.split(",")):
            m = re.fullmatch(r"\s*(\w+)\s*=\s*(-?\d+)\s*", entry)
            if not m:
                raise ImportError(f"{HEADER_PATH}: cannot read the enum entry `{entry.strip()}`")
            constants[m.group(1)] = int(m.group(2))
    constants.update((n, int(v)) for n, v in re.findall(r"^\s*#define\s+(\w+)\s+(-?\d+)\s*$", text, re.M))
    return prototypes, constants


class W2LError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"w2l error {code}: {msg}")
        self.code = code


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU / PyTorch fallback for the hot path)")
    if not os.path.exists(HEADER_PATH):
        raise ImportError(f"{HEADER_PATH} is missing: the signatures of {os.path.basename(LIB_PATH)} are read from it "
                          "(it is part of the source tree)")
    lib = ctypes.CDLL(LIB_PATH)
    with open(HEADER_PATH) as f:
        prototypes, constants = _read_header(f.read())
    for name, (restype, argtypes) in prototypes.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    return lib, prototypes, constants


lib, PROTOTYPES, _constants = _load()
globals().update(_constants)  # W2L_OK, W2L_TERM_ASG, W2L_LN_MAX_PARTS, ...: the names below come from the header

SCALE_MODES = {"none": W2L_SCALE_NONE, "input_sz": W2L_SCALE_INPUT_SZ, "input_sz_sqrt": W2L_SCALE_INPUT_SZ_SQRT,
               "target_sz": W2L_SCALE_TARGET_SZ, "target_sz_sqrt": W2L_SCALE_TARGET_SZ_SQRT}
TERM_FCC, TERM_FAC, TERM_ASG = W2L_TERM_FCC, W2L_TERM_FAC, W2L_TERM_ASG


def _check(rc: int) -> None:
    if rc != 0:
        raise W2LError(rc, lib.w2l_last_error().decode())


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _req(t, dtype, name):
    if t is None:
        return None
    if not t.is_cuda or t.dtype != dtype or not t.is_contiguous():
        raise TypeError(f"{name}: expected a contiguous CUDA tensor of {dtype}")
    return t


_ws_cache: dict = {}


def workspace(nbytes: int, device) -> torch.Tensor:
    key = (str(device), "ws")
    t = _ws_cache.get(key)
    if t is None or t.numel() < nbytes:
        t = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=device)
        _ws_cache[key] = t
    return t


def _mode(m) -> int:
    return SCALE_MODES[m] if isinstance(m, str) else int(m)


def launch_count() -> int:
    return int(lib.w2l_launch_count())


def reset_launch_count() -> None:
    lib.w2l_reset_launch_count()


def set_profile_events(start=None, stop=None) -> None:
    """torch.cuda.Event(enable_timing=True) pair recorded around each call's dominant kernel."""
    if start is None:
        lib.w2l_set_profile_events(None, None)
    else:
        start.record()  # make sure the lazily created handles exist
        stop.record()
        lib.w2l_set_profile_events(ctypes.c_void_p(start.cuda_event), ctypes.c_void_p(stop.cuda_event))


def asg_forward_backward(emis, target, trans, scale_mode="none", dloss=None, terms=TERM_ASG, need_grad=True,
                         out=None, ws=None):
    """Fused ASG (FCC - FAC) forward+backward.  emis [B,T,N] f32, target [B,L] i32 (-1 padded),
    trans [N,N] f32.  Returns (loss[B], d_emis[B,T,N] | None, d_trans[N,N] | None).  N <= 32."""
    return _asg(lib.w2l_asg_workspace_size, lib.w2l_asg_forward_backward, emis, target, trans, scale_mode, dloss,
                terms, need_grad, out, ws)


def asg64_forward_backward(emis, target, trans, scale_mode="none", dloss=None, terms=TERM_ASG, need_grad=True,
                           out=None, ws=None):
    """asg_forward_backward for 1 <= N <= 64 (w2l_asg64_forward_backward)."""
    return _asg(lib.w2l_asg64_workspace_size, lib.w2l_asg64_forward_backward, emis, target, trans, scale_mode, dloss,
                terms, need_grad, out, ws)


def _asg(ws_size, call, emis, target, trans, scale_mode, dloss, terms, need_grad, out, ws):
    emis = _req(emis, torch.float32, "emis")
    trans = _req(trans, torch.float32, "trans")
    target = _req(target, torch.int32, "target")
    dloss = _req(dloss, torch.float32, "dloss")
    B, T, N = emis.shape
    L = 0 if target is None else target.shape[1]
    if out is None:
        loss = torch.empty(B, dtype=torch.float32, device=emis.device)
        d_emis = torch.empty_like(emis) if need_grad else None
        d_trans = torch.empty_like(trans) if need_grad else None
    else:
        loss, d_emis, d_trans = out
    need = ws_size(B, T, N, L)
    if ws is None:
        ws = workspace(need, emis.device)
    _check(call(_stream(), terms, B, T, N, L, _mode(scale_mode), _ptr(emis), _ptr(target),
                _ptr(trans), _ptr(dloss), _ptr(loss), _ptr(d_emis), _ptr(d_trans),
                _ptr(ws), ws.numel()))
    return loss, d_emis, d_trans


def prelu_fwd(x, a, dropout_p=0.0, seed=0):
    """PReLU with one parameter and the fused dropout (the `PR` opcode's kernel): x CUDA float32, a CUDA float32 [1]."""
    x = _req(x, torch.float32, "x")
    a = _req(a, torch.float32, "a")
    y = torch.empty_like(x)
    _check(lib.w2l_prelu_fwd(_stream(), x.numel(), _ptr(x), _ptr(a), _ptr(y), float(dropout_p), int(seed)))
    return y


def prelu_bwd(x, dy, a, dropout_p=0.0, seed=0):
    """(dx, da [1]) of prelu_fwd for the upstream gradient dy; the dropout mask is regenerated from seed."""
    x = _req(x, torch.float32, "x")
    dy = _req(dy, torch.float32, "dy")
    a = _req(a, torch.float32, "a")
    dx = torch.empty_like(x)
    da = torch.empty(1, dtype=torch.float32, device=x.device)
    _check(lib.w2l_prelu_bwd(_stream(), x.numel(), _ptr(x), _ptr(dy), _ptr(a), _ptr(dx), _ptr(da), float(dropout_p), int(seed)))
    return dx, da


def fcc_viterbi(emis, trans):
    """Max-plus FCC Viterbi path [B,T] i32, N <= 32."""
    return _fcc_viterbi(lib.w2l_fcc_viterbi_workspace_size, lib.w2l_fcc_viterbi, emis, trans)


def fcc_viterbi64(emis, trans):
    """fcc_viterbi for 1 <= N <= 64 (w2l_fcc_viterbi64), bit-exact like it."""
    return _fcc_viterbi(lib.w2l_fcc_viterbi64_workspace_size, lib.w2l_fcc_viterbi64, emis, trans)


def _fcc_viterbi(ws_size, call, emis, trans):
    emis = _req(emis, torch.float32, "emis")
    trans = _req(trans, torch.float32, "trans")
    B, T, N = emis.shape
    path = torch.empty((B, T), dtype=torch.int32, device=emis.device)
    ws = workspace(ws_size(B, T, N), emis.device)
    _check(call(_stream(), B, T, N, _ptr(emis), _ptr(trans), _ptr(path), _ptr(ws), ws.numel()))
    return path


def fac_viterbi(emis, target, trans, return_index=False):
    emis = _req(emis, torch.float32, "emis")
    trans = _req(trans, torch.float32, "trans")
    target = _req(target, torch.int32, "target")
    B, T, N = emis.shape
    L = target.shape[1]
    path = torch.empty((B, T), dtype=torch.int32, device=emis.device)
    idx = torch.empty((B, T), dtype=torch.int32, device=emis.device) if return_index else None
    ws = workspace(lib.w2l_fac_viterbi_workspace_size(B, T, N, L), emis.device)
    _check(lib.w2l_fac_viterbi(_stream(), B, T, N, L, _ptr(emis), _ptr(target), _ptr(trans), _ptr(path), _ptr(idx),
                               _ptr(ws), ws.numel()))
    return (path, idx) if return_index else path


def ctc_forward_backward(emis, target, scale_mode="none", dloss=None, need_grad=True, out=None, ws=None, path=None):
    """CTC on raw activations (blank = N-1).  Returns (loss[B], d_emis | None).  path: None, or a CUDA int32 [B, T] tensor
    that receives the per-frame argmax (argmax_path's bits) from the loss's own pass over the activations."""
    emis = _req(emis, torch.float32, "emis")
    target = _req(target, torch.int32, "target")
    dloss = _req(dloss, torch.float32, "dloss")
    path = _req(path, torch.int32, "path")
    B, T, N = emis.shape
    if path is not None and tuple(path.shape) != (B, T):
        raise ValueError(f"path: expected [{B}, {T}], got {tuple(path.shape)}")
    L = 0 if target is None else target.shape[1]
    if out is None:
        loss = torch.empty(B, dtype=torch.float32, device=emis.device)
        d_emis = torch.empty_like(emis) if need_grad else None
    else:
        loss, d_emis = out
    need = lib.w2l_ctc_workspace_size(B, T, N, L)
    if ws is None:
        ws = workspace(need, emis.device)
    if path is None:
        _check(lib.w2l_ctc_forward_backward(_stream(), B, T, N, L, _mode(scale_mode), _ptr(emis), _ptr(target),
                                            _ptr(dloss), _ptr(loss), _ptr(d_emis), _ptr(ws), ws.numel()))
    else:
        _check(lib.w2l_ctc_forward_backward_path(_stream(), B, T, N, L, _mode(scale_mode), _ptr(emis), _ptr(target),
                                                 _ptr(dloss), _ptr(loss), _ptr(d_emis), _ptr(path), _ptr(ws), ws.numel()))
    return loss, d_emis


def argmax_path(emis):
    emis = _req(emis, torch.float32, "emis")
    B, T, N = emis.shape
    path = torch.empty((B, T), dtype=torch.int32, device=emis.device)
    _check(lib.w2l_argmax_path(_stream(), B, T, N, _ptr(emis), _ptr(path)))
    return path


def ctc_viterbi_target(emis, target, return_state=False):
    """CTC forced alignment on raw activations (blank = N-1): path [B,T] int32 (label or blank per frame, -1 for a
    target that cannot be aligned) and, with return_state, the extended-target state per frame."""
    emis = _req(emis, torch.float32, "emis")
    target = _req(target, torch.int32, "target")
    B, T, N = emis.shape
    L = target.shape[1]
    path = torch.empty((B, T), dtype=torch.int32, device=emis.device)
    state = torch.empty((B, T), dtype=torch.int32, device=emis.device) if return_state else None
    ws = workspace(lib.w2l_ctc_viterbi_workspace_size(B, T, N, L), emis.device)
    _check(lib.w2l_ctc_viterbi_target(_stream(), B, T, N, L, _ptr(emis), _ptr(target), _ptr(path), _ptr(state), _ptr(ws),
                                      ws.numel()))
    return (path, state) if return_state else path


def linseg_target(target, T: int):
    target = _req(target, torch.int32, "target")
    B, L = target.shape
    out = torch.empty((B, int(T)), dtype=torch.int32, device=target.device)
    _check(lib.w2l_linseg_target(_stream(), B, int(T), L, _ptr(target), _ptr(out)))
    return out


class ProfileList:
    """n CUDA event pairs recorded around the dominant-kernel launches of `kind` (1 GEMM, 2 criterion chains)."""

    def __init__(self, kind: int, n: int):
        self.starts = [torch.cuda.Event(enable_timing=True) for _ in range(n)]
        self.stops = [torch.cuda.Event(enable_timing=True) for _ in range(n)]
        for e in self.starts + self.stops:
            e.record()
        self._a = (ctypes.c_void_p * n)(*[e.cuda_event for e in self.starts])
        self._b = (ctypes.c_void_p * n)(*[e.cuda_event for e in self.stops])
        self.kind, self.n = kind, n

    def arm(self):
        lib.w2l_set_profile_event_list(self.kind, self._a, self._b, self.n)

    def disarm(self) -> int:
        used = int(lib.w2l_profile_events_used())
        lib.w2l_set_profile_event_list(0, None, None, 0)
        return used

    def times_ms(self, used: int):
        return [self.starts[k].elapsed_time(self.stops[k]) for k in range(used)]


def trace_list() -> list:
    """every launch of the last trace() in order: [(kernel name, ms)]"""
    buf = ctypes.create_string_buffer(1 << 18)
    lib.w2l_trace_list(buf, len(buf))
    return [(ln.split("\t")[0], float(ln.split("\t")[1])) for ln in buf.value.decode().splitlines()]


PRECISIONS = {"tf32": W2L_PRECISION_TF32, "f32": W2L_PRECISION_F32, "fp32": W2L_PRECISION_F32, "bf16": W2L_PRECISION_BF16,
              "fp16": W2L_PRECISION_FP16}
GEMM_KINDS = {"tf32": W2L_GEMM_TF32, "f32x3": W2L_GEMM_F32X3, "bf16": W2L_GEMM_BF16, "f32x3_split_b": W2L_GEMM_F32X3_SPLIT_B,
              "fp16": W2L_GEMM_FP16}


def set_precision(p) -> None:
    """tf32 (default) | f32 (fp32-accurate 3xTF32 GEMMs and mma.sync time convolutions) | bf16 (bf16 GEMM operands) |
    fp16 (fp16 GEMM operands)."""
    _check(lib.w2l_set_precision(PRECISIONS[p] if isinstance(p, str) else int(p)))


def get_precision() -> int:
    return int(lib.w2l_get_precision())


def gemm(A, B, kind="tf32", a_mn=False, b_mn=False, bias=None, act=0, out=None, out_bf16=False, accumulate=False, aux=None,
         aux_mode=0, aux_scale=1.0, dropout_p=0.0, seed=0, M=None, N=None, K=None, lda=None, ldb=None, allow_overlap=False):
    """General wgmma GEMM (w2l_gemm): A/B fp32 (kinds tf32, f32x3), bfloat16 (kind bf16) or float16 (kind fp16); C fp32 or
    16-bit (out_bf16: float16 for kind fp16, bfloat16 otherwise), aux likewise.
    Kind f32x3_split_b: B is the [2][N][ldb] planes of split_tf32 (K is taken from A)."""
    if M is None:
        M, K = (A.shape[1], A.shape[0]) if a_mn else A.shape
        N = B.shape[-2] if B.dim() == 3 else (B.shape[1] if b_mn else B.shape[0])
    lda = A.stride(0) if lda is None else lda
    ldb = B.stride(-2) if ldb is None else ldb
    kind_id = GEMM_KINDS[kind] if isinstance(kind, str) else int(kind)
    half = torch.float16 if kind_id == GEMM_KINDS["fp16"] else torch.bfloat16  # the kind's 16-bit C / aux type
    if out is None:
        out = torch.empty((M, N), dtype=half if out_bf16 else torch.float32, device=A.device)
    if out.dtype not in (torch.float32, half) or (aux is not None and aux.dtype not in (torch.float32, half)):
        raise TypeError(f"gemm: a 16-bit C or aux of kind {kind} is {half}")
    _check(lib.w2l_gemm(_stream(), kind_id, int(a_mn), int(b_mn), M, N, K, _ptr(A), lda, _ptr(B), ldb, _ptr(out),
                        out.stride(0), int(out.dtype == half), _ptr(bias), int(act), int(accumulate), _ptr(aux),
                        0 if aux is None else aux.stride(0), int(aux is not None and aux.dtype == half),
                        int(aux_mode), float(aux_scale), float(dropout_p), int(seed), int(allow_overlap)))
    return out


def cast_bf16(x):
    x = _req(x, torch.float32, "x")
    y = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    _check(lib.w2l_cast_bf16(_stream(), x.numel(), _ptr(x), _ptr(y)))
    return y


def cast_fp16(x):
    x = _req(x, torch.float32, "x")
    y = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    _check(lib.w2l_cast_fp16(_stream(), x.numel(), _ptr(x), _ptr(y)))
    return y


def cast_fp16_rows(x, cols_padded):
    """rows of a 2-D fp32 tensor (rows contiguous) -> [rows][cols_padded] float16, zero-padded columns"""
    x = _req(x, torch.float32, "x")
    if x.dim() != 2 or x.stride(1) != 1:
        raise TypeError("cast_fp16_rows: x must be 2-D with contiguous rows")
    y = torch.empty((x.shape[0], cols_padded), dtype=torch.float16, device=x.device)
    _check(lib.w2l_cast_fp16_rows(_stream(), x.shape[0], x.shape[1], x.stride(0), cols_padded, _ptr(x), _ptr(y)))
    return y


def split_tf32(x, transpose=False, cols_padded=None):
    """B planes of kind f32x3_split_b from a 2-D fp32 tensor x (rows contiguous): [2][rows][cols_padded] tf32 hi / lo,
    or with transpose those of x^T, [2][cols][cols_padded]; cols_padded defaults to the source row length rounded up
    to 4 (a TMA row)"""
    if x.dtype != torch.float32 or not x.is_cuda or x.dim() != 2 or x.stride(1) != 1:
        raise TypeError("split_tf32: x must be a 2-D CUDA float32 tensor with contiguous rows")
    rows, cols = x.shape
    k = rows if transpose else cols
    cols_padded = (k + 3) // 4 * 4 if cols_padded is None else cols_padded
    y = torch.empty((2, cols if transpose else rows, cols_padded), dtype=torch.float32, device=x.device)
    _check(lib.w2l_split_tf32(_stream(), int(transpose), rows, cols, x.stride(0), cols_padded, _ptr(x), _ptr(y)))
    return y


def gemm_set_variant(v: int = 1):
    """1: one CTA per SM walking the tiles (default); 0: one tile per CTA"""
    _check(lib.w2l_gemm_set_variant(int(v)))


def gemm_set_tile(bn: int = 0):
    _check(lib.w2l_gemm_set_tile(int(bn)))


def trace(fn, capacity: int = 4096) -> dict:
    """Run fn() (all work on the current stream) in trace mode; returns {kernel name: (launches, total ms)} measured
    with one CUDA event after every launch — the warm, in-situ share of each kernel (measurement only)."""
    _check(lib.w2l_trace_begin(_stream(), capacity))
    try:
        fn()
    finally:
        buf = ctypes.create_string_buffer(1 << 16)
        lib.w2l_trace_end(buf, len(buf))
    out = {}
    for line in buf.value.decode().splitlines():
        name, n, ms = line.split("\t")
        out[name] = (int(n), float(ms))
    return out


def gemm_tf32(A, B, bias=None, act=0, a_mn=False, b_mn=False, out=None):
    """C[m][n] = act(sum_k A(m,k) B(n,k) + bias[n]).  A: [M,K] (or [K,M] if a_mn), B: [N,K] (or [K,N] if b_mn)."""
    A = _req(A, torch.float32, "A")
    B = _req(B, torch.float32, "B")
    bias = _req(bias, torch.float32, "bias")
    M, K = (A.shape[1], A.shape[0]) if a_mn else A.shape
    N = B.shape[1] if b_mn else B.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=A.device)
    _check(lib.w2l_gemm_tf32(_stream(), int(a_mn), int(b_mn), M, N, K, _ptr(A), A.stride(0), _ptr(B), B.stride(0),
                             _ptr(out), out.stride(0), _ptr(bias), int(act)))
    return out


def gemm_tf32_ex(A, B, out, bias=None, act=0, a_mn=False, b_mn=False, accumulate=False, aux=None, aux_mode=0,
                 aux_scale=1.0, dropout_p=0.0, seed=0):
    M, K = (A.shape[1], A.shape[0]) if a_mn else A.shape
    N = B.shape[1] if b_mn else B.shape[0]
    _check(lib.w2l_gemm_tf32_ex(_stream(), int(a_mn), int(b_mn), M, N, K, _ptr(A), A.stride(0), _ptr(B), B.stride(0),
                                _ptr(out), out.stride(0), _ptr(bias), int(act), int(accumulate), _ptr(aux),
                                0 if aux is None else aux.stride(0), int(aux_mode), float(aux_scale), float(dropout_p),
                                int(seed)))
    return out


def gemm_tf32_view(A, lda, B, ldb, out, M, N, K, a_mn=False, b_mn=False, bias=None, act=0, accumulate=False):
    """GEMM on raw (possibly overlapping-row) operand views: A/B are any CUDA float tensors, lda/ldb explicit."""
    _check(lib.w2l_gemm_tf32_view(_stream(), int(a_mn), int(b_mn), M, N, K, _ptr(A), lda, _ptr(B), ldb, _ptr(out), out.stride(0),
                                  _ptr(bias), int(act), int(accumulate)))
    return out


def conv_time_ws(B, Tout, Cin, Cout, K, device):
    return workspace(lib.w2l_conv_time_workspace_size(B, Tout, Cin, Cout, K), device)


def conv_time_fwd(x, wt, bias, Tout, stride, pad_left, act=0, dropout_p=0.0, seed=0, add=None):
    """x [B,T,Cin,W], wt [Cout,Cin,K] -> y [B,Tout,Cout,W]"""
    B, T, Cin, W = x.shape
    Cout, _, K = wt.shape
    y = torch.empty((B, Tout, Cout, W), dtype=torch.float32, device=x.device)
    ws = conv_time_ws(B, Tout, Cin, Cout, K, x.device)
    _check(lib.w2l_conv_time_fwd(_stream(), B, T, Tout, W, Cin, Cout, K, stride, pad_left, _ptr(x), _ptr(wt), _ptr(bias),
                                 _ptr(add), _ptr(y), act, float(dropout_p), int(seed), _ptr(ws), ws.numel()))
    return y


def conv_time_dgrad(dy, wt, T, stride, pad_left, add=None, out=None):
    """dx = conv^T(dy) (+ add); out may be the same tensor as add (in-place accumulation)."""
    B, Tout, Cout, W = dy.shape
    _, Cin, K = wt.shape
    dx = out if out is not None else torch.empty((B, T, Cin, W), dtype=torch.float32, device=dy.device)
    ws = conv_time_ws(B, Tout, Cin, Cout, K, dy.device)
    _check(lib.w2l_conv_time_dgrad(_stream(), B, T, Tout, W, Cin, Cout, K, stride, pad_left, _ptr(dy), _ptr(wt), _ptr(add),
                                   _ptr(dx), _ptr(ws), ws.numel()))
    return dx


def conv_time_wgrad(x, dy, K, stride, pad_left, dwt=None, dbias=None):
    B, T, Cin, W = x.shape
    _, Tout, Cout, _ = dy.shape
    if dwt is None:
        dwt = torch.zeros((Cout, Cin, K), dtype=torch.float32, device=x.device)
        dbias = torch.zeros(Cout, dtype=torch.float32, device=x.device)
    ws = conv_time_ws(B, Tout, Cin, Cout, K, x.device)
    _check(lib.w2l_conv_time_wgrad(_stream(), B, T, Tout, W, Cin, Cout, K, stride, pad_left, _ptr(x), _ptr(dy), _ptr(dwt),
                                   _ptr(dbias), _ptr(ws), ws.numel()))
    return dwt, dbias


def layernorm_scratch(B: int, device) -> torch.Tensor:
    """the scratch of w2l_layernorm_fwd / w2l_layernorm_bwd over B groups: W2L_LN_SCRATCH_DOUBLES(B) float64"""
    return torch.empty(2 * W2L_LN_MAX_PARTS * B, dtype=torch.float64, device=device)


def layernorm_fwd(a, r, gain, bias, eps=1e-5):
    B = a.shape[0]
    R = a[0].numel()
    y = torch.empty_like(a)
    mr = torch.empty((B, 2), dtype=torch.float32, device=a.device)
    scratch = layernorm_scratch(B, a.device)
    _check(lib.w2l_layernorm_fwd(_stream(), B, R, float(eps), _ptr(a), _ptr(r), _ptr(gain), _ptr(bias), _ptr(y), _ptr(mr),
                                 _ptr(scratch)))
    return y, mr


def layernorm_bwd(a, r, dy, gain, mr, branch_mode=0, branch_scale=1.0):
    B = a.shape[0]
    R = a[0].numel()
    d_branch = torch.empty_like(a)
    d_res = torch.empty_like(a)
    dgain = torch.zeros(1, dtype=torch.float32, device=a.device)
    dbias = torch.zeros(1, dtype=torch.float32, device=a.device)
    scratch = layernorm_scratch(B, a.device)
    _check(lib.w2l_layernorm_bwd(_stream(), B, R, _ptr(a), _ptr(r), _ptr(dy), _ptr(gain), _ptr(mr), _ptr(d_branch),
                                 _ptr(d_res), int(branch_mode), float(branch_scale), _ptr(dgain), _ptr(dbias),
                                 _ptr(scratch)))
    return d_branch, d_res, dgain, dbias


def soft_label_loss(student, teacher, scale=1.0, need_grad=True, d_student=None):
    """slimIPL's soft-label loss (w2l_soft_label_loss) over logits [..., N] (rows = every leading index): returns
    (loss float32 [1] = -scale / rows * sum_rows sum_c softmax(teacher)_c logSoftmax(student)_c,
    d_student = scale / rows * (softmax(student) - softmax(teacher)) or None).  d_student: an output buffer of the
    student's shape (any float alignment)."""
    student = _req(student, torch.float32, "student")
    teacher = _req(teacher, torch.float32, "teacher")
    if student.shape != teacher.shape:
        raise ValueError(f"soft_label_loss: teacher shape {tuple(teacher.shape)} != student shape {tuple(student.shape)}")
    N = student.shape[-1]
    rows = student.numel() // N
    loss = torch.empty(1, dtype=torch.float32, device=student.device)
    ws = torch.empty(rows, dtype=torch.float32, device=student.device)
    if need_grad and d_student is None:
        d_student = torch.empty_like(student)
    d = _req(d_student, torch.float32, "d_student") if need_grad else None
    _check(lib.w2l_soft_label_loss(_stream(), rows, N, _ptr(student), _ptr(teacher), float(scale), _ptr(loss), _ptr(d), _ptr(ws)))
    return loss, d


def ema_update(ema, params, decay):
    """in place: ema = ema * decay + params * (1 - decay) (w2l_ema_update), float32 tensors of the same size"""
    ema = _req(ema, torch.float32, "ema")
    params = _req(params, torch.float32, "params")
    if ema.numel() != params.numel():
        raise ValueError("ema_update: sizes differ")
    _check(lib.w2l_ema_update(_stream(), ema.numel(), _ptr(ema), _ptr(params), float(decay)))
    return ema
