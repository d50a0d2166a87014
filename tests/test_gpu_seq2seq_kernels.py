"""The Seq2Seq criterion's kernels (csrc/seq2seq.cu) called one by one through their C entry points, each against a plain
model of its contract in include/w2l_b200.h, at the shapes where the kernels change structure:

- GRU forward and backward (w2l_seq2seq_gru_fwd / _bwd) against a float64 recurrence built on oracle/seq2seq_ref.py's
  GRU step: a partial last CTA (J = ceil(H / SMs) units per CTA, the last one holding fewer), batches that cross the
  forward's and the backward's row chunks with a ragged remainder, U = 1 over hundreds of rows (the decode and the beam
  search), a long recurrence, h0 given and NULL, no stash;
- attention forward and backward, unsized and _sized, against oracle/seq2seq_ref.py's attention in float64: partial
  8-step and 8-frame tiles, T' up to the last frame that fits in shared memory (7040 - H) and U up to 3520 for the
  gradient, one more of either refused with nothing launched, the soft window, per-utterance frame counts with
  NaN-poisoned keys and values past them;
- the loss and scale_rows against float64 log-softmax, and the per-utterance sum against a float32 sum in row order, bit
  for bit;
- the embedding gradient against a NumPy float32 model of its summation order, bit for bit;
- the greedy step's argmax and the beam search's first step against NumPy and tests/seq2seq_beam_reference.py's walk,
  index for index, with heavy exact ties at N = 65 536.

Shapes come from the device's SM count through the kernels' own formulas, and every case asserts that the edge it is
named for is reached on the device it runs on.  Float64 bounds keep a margin of 3-5x over the error measured on an H100
80GB HBM3 (132 SMs); each carries its measured value.  Every check appends its measured error to
w2l_seq2seq_kernels.jsonl in the temporary directory."""
import ctypes
import json
import math
import os
import tempfile

import numpy as np
import pytest
import torch

from oracle.seq2seq_ref import attention, gru_layer, window
from seq2seq_beam_reference import beam

pytestmark = pytest.mark.gpu

# csrc/seq2seq.cu's launch constants
SMEM_LIMIT = 220 * 1024  # bytes of dynamic shared memory a kernel may ask for
BATCH_CHUNK = 16         # most rows the recurrence stages at a time
U_TILE, T_TILE = 8, 8    # decoder steps per attention CTA, frames per attention-gradient CTA
ERR_UNSUPPORTED = 4


def _lib():
    from wav2letter_b200 import capi

    return capi


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _s():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ok(rc):
    capi = _lib()
    assert rc == 0, capi.lib.w2l_last_error().decode()


def _within(name, err, bound):
    """err <= bound, with err appended to the measurement log"""
    with open(os.path.join(tempfile.gettempdir(), "w2l_seq2seq_kernels.jsonl"), "a") as f:
        f.write(json.dumps({"check": name, "err": err, "bound": bound}) + "\n")
    assert err <= bound, f"{name}: error {err:.3g} above the bound {bound:.3g}"


def rel(a, b):
    """max |a - b| / max |b| over the whole tensor"""
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- the recurrence's schedule, by the kernel's own formulas --------------------------------------------------------
def gru_units(H):
    return -(-H // sms())


def gru_last_units(H):
    """units of the last CTA (fewer than J: a partial CTA)"""
    J = gru_units(H)
    return H - (-(-H // J) - 1) * J


def gru_chunk(fixed, per_row):
    bc = BATCH_CHUNK
    while bc >= 1:
        if 4 * (fixed + bc * per_row) <= SMEM_LIMIT:
            return bc
        bc //= 2
    return 0


def gru_fwd_chunk(H):
    J = gru_units(H)
    return gru_chunk(3 * J * H, H + 3 * J)


def gru_bwd_chunk(H):
    J = gru_units(H)
    return gru_chunk(3 * J * H, 3 * H + J)


def partial_hs():
    """every H the kernels take whose last CTA is partial"""
    return [H for H in range(32, 1025, 32) if gru_last_units(H) < gru_units(H)]


def gru_ref(gi, Whh, bhh, h0):
    """float64 recurrence from the input projection gi [B,U,3H] (oracle/seq2seq_ref.py's gru_layer step with
    gi = x W_ih^T + b_ih precomputed): outputs [B,U,H], the stash planes [5][B,U,H] and every step's gh = W_hh h + b_hh
    (retained, for its gradient)"""
    B, U, H3 = gi.shape
    H = H3 // 3
    h = torch.zeros(B, H, dtype=gi.dtype, device=gi.device) if h0 is None else h0
    outs, planes, ghs = [], [], []
    for u in range(U):
        gh = h @ Whh.T + bhh
        if gh.requires_grad:
            gh.retain_grad()
        ghs.append(gh)
        r = torch.sigmoid(gi[:, u, :H] + gh[:, :H])
        z = torch.sigmoid(gi[:, u, H:2 * H] + gh[:, H:2 * H])
        n = torch.tanh(gi[:, u, 2 * H:] + r * gh[:, 2 * H:])
        planes.append(torch.stack([r, z, n, gh[:, 2 * H:], h]))
        h = (1 - z) * n + z * h
        outs.append(h)
    return torch.stack(outs, 1), torch.stack(planes, 2), ghs


def test_gru_ref_is_the_oracle_layer():
    g = torch.Generator().manual_seed(1)
    B, U, H = 3, 5, 8
    x, h0 = torch.randn(B, U, H, generator=g, dtype=torch.float64), torch.randn(B, H, generator=g, dtype=torch.float64)
    W_ih, W_hh = (torch.randn(3 * H, H, generator=g, dtype=torch.float64) / math.sqrt(H) for _ in range(2))
    b_ih, b_hh = (torch.randn(3 * H, generator=g, dtype=torch.float64) for _ in range(2))
    want, _ = gru_layer(x, W_ih, W_hh, b_ih, b_hh, h0)
    got, _, _ = gru_ref((x @ W_ih.T + b_ih).requires_grad_(True), W_hh, b_hh, h0)
    assert torch.allclose(got, want, rtol=0, atol=1e-14)


# Errors against float64 (max |error| / max |reference| per tensor), measured on an H100 80GB HBM3 (132 SMs) as the largest
# over the cases below; the bounds keep 3.4x or more.  The 300-step recurrence measured no growth: 2.2e-7 on out,
# 2.1e-7 on dgh.
GRU_TOL = {
    "out": 1.0e-6,      # measured 2.2e-7
    "stash": 1.0e-6,    # measured 3.0e-7 (n)
    "dgi": 1.0e-6,      # measured 2.5e-7
    "dgh": 1.0e-6,      # measured 2.9e-7
}


def gru_case(case):
    """(B, U, H, h0 given) of a named case, and the edges it must reach"""
    hs = partial_hs()
    assert len(hs) >= 2, f"no two H with a partial last CTA on {sms()} SMs"
    if case == "partial_small":
        return 5, 12, hs[0], True
    if case == "partial_large":  # also one row more than the backward's chunk
        return gru_bwd_chunk(hs[-1]) + 1, 10, hs[-1], False
    if case == "chunks_9":
        return 9, 6, 1024, True
    if case == "chunks_41":
        return 41, 4, 1024, False
    if case == "decode_rows":
        return 512, 1, 512, True
    if case == "long":
        return 3, 300, hs[0], False
    raise KeyError(case)


@pytest.mark.parametrize("case", ["partial_small", "partial_large", "chunks_9", "chunks_41", "decode_rows", "long"])
def test_gru_fwd_bwd(case):
    lib = _lib().lib
    B, U, H, with_h0 = gru_case(case)
    J, BCf, BCb = gru_units(H), gru_fwd_chunk(H), gru_bwd_chunk(H)
    if case.startswith("partial"):
        assert gru_last_units(H) < J, (H, J)
    if case.startswith("chunks"):  # more rows than the backward's chunk, with a ragged last chunk
        assert BCb < BCf and B > BCb and B % BCb, (B, BCf, BCb)
    if case == "chunks_41":  # the forward's too
        assert B > BCf and B % BCf, (B, BCf)

    g = torch.Generator(device="cuda").manual_seed(H * 1000 + B * 10 + U)
    gi = torch.randn(B * U, 3 * H, device="cuda", generator=g)
    Whh = torch.randn(3 * H, H, device="cuda", generator=g) / math.sqrt(H)
    bhh = torch.randn(3 * H, device="cuda", generator=g) * 0.5
    h0 = torch.randn(B, H, device="cuda", generator=g) * 0.5 if with_h0 else None
    dout = torch.randn(B * U, H, device="cuda", generator=g)

    assert lib.w2l_seq2seq_gru_stash_floats(B, U, H) == 5 * B * U * H
    out = torch.full((B * U, H), float("nan"), device="cuda")
    stash = torch.full((5, B * U, H), float("nan"), device="cuda")
    _ok(lib.w2l_seq2seq_gru_fwd(_s(), B, U, H, _p(gi), _p(Whh), _p(bhh), _p(h0), _p(out), _p(stash)))
    out_nostash = torch.full((B * U, H), float("nan"), device="cuda")
    _ok(lib.w2l_seq2seq_gru_fwd(_s(), B, U, H, _p(gi), _p(Whh), _p(bhh), _p(h0), _p(out_nostash), None))
    dgi = torch.full((B * U, 3 * H), float("nan"), device="cuda")
    dgh = torch.full((B * U, 3 * H), float("nan"), device="cuda")
    carry = torch.full((B, H), float("nan"), device="cuda")
    _ok(lib.w2l_seq2seq_gru_bwd(_s(), B, U, H, _p(dout), _p(Whh), _p(stash), _p(dgi), _p(dgh), _p(carry)))
    assert torch.equal(out_nostash, out), "the stash changes the outputs"

    gi64 = gi.double().view(B, U, 3 * H).requires_grad_(True)
    bhh64 = bhh.double().requires_grad_(True)  # every step's gh then carries a gradient
    ref, planes, ghs = gru_ref(gi64, Whh.double(), bhh64, None if h0 is None else h0.double())
    (ref * dout.double().view(B, U, H)).sum().backward()
    tol = GRU_TOL
    _within(f"gru.{case}.out", rel(out, ref.detach().reshape(B * U, H)), tol["out"])
    for k, name in enumerate(["r", "z", "n", "gh_n", "h_prev"]):
        _within(f"gru.{case}.stash.{name}", rel(stash[k], planes[k].detach().reshape(B * U, H)), tol["stash"])
    _within(f"gru.{case}.dgi", rel(dgi, gi64.grad.reshape(B * U, 3 * H)), tol["dgi"])
    dgh_ref = torch.stack([gh.grad for gh in ghs], 1).reshape(B * U, 3 * H)
    _within(f"gru.{case}.dgh", rel(dgh, dgh_ref), tol["dgh"])


# ---- attention ------------------------------------------------------------------------------------------------------
def attn_max_frames(H):
    """the most encoder frames the attention stages: 8 (H + T') floats of shared memory"""
    return SMEM_LIMIT // (4 * U_TILE) - H


def attn_max_steps():
    """the most decoder steps the attention gradient stages: 2 * 8 U floats"""
    return SMEM_LIMIT // (4 * 2 * T_TILE)


def window_ref(U, Tb, Ub, std):
    """w[u][t] = -(t - u T'_b / U_b)^2 / (2 std^2), t < T'_b, in fp32: the centre (float)u * (float)T'_b / (float)U_b as
    DESIGN.md §9 fixes it, then -(d d) fp32(1 / (2 std^2)) as the kernel evaluates it.  Against a float64 window, the fp32 centre
    alone moves the weights by 1.3e-6 at T' = 1000, where u T' / U is not a whole number."""
    u = np.arange(U, dtype=np.float32)[:, None]
    c = (u * np.float32(Tb)) / np.float32(Ub)
    d = np.arange(Tb, dtype=np.float32)[None, :] - c
    return torch.from_numpy((-(d * d) * np.float32(1.0 / (2.0 * std * std))).astype(np.float64))


def test_window_ref_is_the_oracle_window():
    """where fp32 is exact, the window is oracle/seq2seq_ref.py's"""
    assert torch.equal(window_ref(8, 24, 8, 2.0), window(8, 24, 2.0))


def attn_ref(q, x, tps, ups, std):
    """float64 out, weights and the gradients of sum(out * dout) per utterance, over its first T'_b frames"""
    B, U, H = q.shape
    q64 = q.double().requires_grad_(True)
    x64 = x.double().nan_to_num(0.0).requires_grad_(True)
    outs, ws = [], []
    for b in range(B):
        Tb = tps[b]
        xb = x64[b:b + 1, :Tb]
        win = window_ref(U, Tb, ups[b], std).to(q.device) if std > 0 else None
        k = xb[..., :H]
        s = q64[b:b + 1] @ k.transpose(1, 2) / math.sqrt(H)
        if win is not None:
            s = s + win
        w = torch.zeros(1, U, x.shape[1], dtype=torch.float64, device=q.device)
        w[..., :Tb] = torch.softmax(s, -1)
        ws.append(w.detach())
        outs.append(attention(q64[b:b + 1], xb, win))
    return q64, x64, torch.cat(outs), torch.cat(ws)


# Errors against float64 (max |error| / max |reference|; absolute on the weights, which are in [0, 1]), measured on an
# H100 80GB HBM3 as the largest over the tile cases and the frame limits; the bounds keep about 4x.
ATTN_TOL = {
    "out": 7.0e-7,      # measured 1.8e-7
    "attn": 1.0e-6,     # measured 2.2e-7
    "dq": 7.0e-7,       # measured 1.9e-7
    "dx": 1.5e-6,       # measured 3.6e-7
}
# The step limit's second utterance has U_b = 700 of U = 3520 steps over T'_b = 13 frames: on the rows past U_b the
# window's centre lies up to 52 frames past the last one, so the softmax takes scores s + w of magnitude ~100 whose fp32
# rounding (|s + w| eps) moves the weights by ~1e-6 in any fp32 evaluation.  Measured there, the bounds keep about 4x.
ATTN_FAR_WINDOW_TOL = {
    "out": 3.0e-6,      # measured 7.4e-7
    "attn": 5.0e-6,     # measured 1.3e-6
    "dq": 5.0e-6,       # measured 1.2e-6
    "dx": 7.0e-6,       # measured 1.7e-6
}


def run_attn(name, B, U, Tp, H, tps, ups, std, seed, tol=ATTN_TOL):
    """the forward and the backward (sized when tps is given), checked against float64; keys and values past T'_b are NaN"""
    lib = _lib().lib
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(B, U, H, device="cuda", generator=g)
    x = torch.randn(B, Tp, 2 * H, device="cuda", generator=g)
    dout = torch.randn(B, U, H, device="cuda", generator=g)
    sized = tps is not None
    tp = tps if sized else [Tp] * B
    up = ups if ups is not None else [U] * B
    for b in range(B):
        x[b, tp[b]:] = float("nan")
    out = torch.full((B, U, H), float("nan"), device="cuda")
    attn = torch.full((B, U, Tp), float("nan"), device="cuda")
    dq = torch.full((B, U, H), float("nan"), device="cuda")
    dx = torch.full((B, Tp, 2 * H), float("nan"), device="cuda")
    dS = torch.full((B, U, Tp), float("nan"), device="cuda")
    if sized:
        tps_d = torch.tensor(tps, dtype=torch.int32, device="cuda")
        ups_d = None if ups is None else torch.tensor(ups, dtype=torch.int32, device="cuda")
        _ok(lib.w2l_seq2seq_attn_fwd_sized(_s(), B, U, Tp, H, _p(q), _p(x), _p(tps_d), _p(ups_d), U, std, _p(out), _p(attn)))
        _ok(lib.w2l_seq2seq_attn_bwd_sized(_s(), B, U, Tp, H, _p(q), _p(x), _p(attn), _p(dout), _p(tps_d), _p(dq), _p(dx), _p(dS)))
    else:
        _ok(lib.w2l_seq2seq_attn_fwd(_s(), B, U, Tp, H, _p(q), _p(x), U, std, _p(out), _p(attn)))
        _ok(lib.w2l_seq2seq_attn_bwd(_s(), B, U, Tp, H, _p(q), _p(x), _p(attn), _p(dout), _p(dq), _p(dx), _p(dS)))
    for t in (out, attn, dq, dx):
        assert not t.isnan().any(), f"{name}: NaN in a result"
    for b in range(B):
        assert torch.all(attn[b, :, tp[b]:] == 0) and torch.all(dx[b, tp[b]:] == 0), f"{name}: nonzero past T'_b"
    q64, x64, ref, wref = attn_ref(q, x, tp, up, std)
    (ref * dout.double()).sum().backward()
    _within(f"attn.{name}.out", rel(out, ref.detach()), tol["out"])
    _within(f"attn.{name}.attn", float((attn.double() - wref).abs().max()), tol["attn"])
    _within(f"attn.{name}.dq", rel(dq, q64.grad), tol["dq"])
    _within(f"attn.{name}.dx", rel(dx, x64.grad), tol["dx"])


@pytest.mark.parametrize("Tp", [1, 2, 9, 1000])
@pytest.mark.parametrize("U", [1, 7, 8, 9])
def test_attention_tiles(U, Tp):
    H = 64
    for std in (0.0, 4.0):
        run_attn(f"U{U}.T{Tp}.w{std:g}", 2, U, Tp, H, None, None, std, U * 10007 + Tp)
    # per-utterance frame counts: all T', a single frame, about half and one short; target sizes at and below U
    tps = [Tp, 1, max(1, (Tp + 1) // 2), max(1, Tp - 1)]
    ups = [U, max(1, U - 2), 1, U]
    for std in (0.0, 4.0):
        run_attn(f"U{U}.T{Tp}.w{std:g}.sized", 4, U, Tp, H, tps, ups, std, U * 10007 + Tp + 1)


@pytest.mark.parametrize("H", [32, 512, 1024])
def test_attention_frame_limit(H):
    """the last T' that fits in shared memory runs and is right; one frame more is refused and launches nothing"""
    capi = _lib()
    lib = capi.lib
    Tmax = attn_max_frames(H)
    assert 4 * U_TILE * (H + Tmax) <= SMEM_LIMIT < 4 * U_TILE * (H + Tmax + 1)
    hit = capi.trace(lambda: run_attn(f"limit.H{H}", 2, 9, Tmax, H, [Tmax, Tmax - 5], None, 40.0, H))
    assert "seq2seq_attn_fwd_kernel" in hit and "seq2seq_attn_bwd_kv_kernel" in hit, hit
    T = Tmax + 1
    B, U = 1, 9
    q = torch.zeros(B, U, H, device="cuda")
    x = torch.zeros(B, T, 2 * H, device="cuda")
    out, dq = torch.zeros_like(q), torch.zeros_like(q)
    attn, dS = torch.zeros(B, U, T, device="cuda"), torch.zeros(B, U, T, device="cuda")
    dx = torch.zeros_like(x)
    tps = torch.full((B,), T, dtype=torch.int32, device="cuda")
    rcs = []
    launched = capi.trace(lambda: rcs.extend([
        lib.w2l_seq2seq_attn_fwd(_s(), B, U, T, H, _p(q), _p(x), U, 0.0, _p(out), _p(attn)),
        lib.w2l_seq2seq_attn_fwd_sized(_s(), B, U, T, H, _p(q), _p(x), _p(tps), None, U, 0.0, _p(out), _p(attn)),
        lib.w2l_seq2seq_attn_bwd(_s(), B, U, T, H, _p(q), _p(x), _p(attn), _p(q), _p(dq), _p(dx), _p(dS)),
        lib.w2l_seq2seq_attn_bwd_sized(_s(), B, U, T, H, _p(q), _p(x), _p(attn), _p(q), _p(tps), _p(dq), _p(dx), _p(dS)),
    ]))
    assert rcs == [ERR_UNSUPPORTED] * 4 and launched == {}, (rcs, launched)


def test_attention_step_limit():
    """the gradient stages 2 * 8 U floats: U = 3520 runs and is right, U = 3521 is refused and launches nothing"""
    capi = _lib()
    lib = capi.lib
    Umax = attn_max_steps()
    assert 4 * 2 * T_TILE * Umax <= SMEM_LIMIT < 4 * 2 * T_TILE * (Umax + 1)
    run_attn("limit.U", 2, Umax, 21, 32, [21, 13], [Umax, 700], 4.0, 7, ATTN_FAR_WINDOW_TOL)
    B, U, T, H = 1, Umax + 1, 21, 32
    q, dq = torch.zeros(B, U, H, device="cuda"), torch.zeros(B, U, H, device="cuda")
    x, dx = torch.zeros(B, T, 2 * H, device="cuda"), torch.zeros(B, T, 2 * H, device="cuda")
    attn, dS = torch.zeros(B, U, T, device="cuda"), torch.zeros(B, U, T, device="cuda")
    rcs = []
    launched = capi.trace(lambda: rcs.extend([
        lib.w2l_seq2seq_attn_bwd(_s(), B, U, T, H, _p(q), _p(x), _p(attn), _p(q), _p(dq), _p(dx), _p(dS)),
        lib.w2l_seq2seq_attn_bwd_sized(_s(), B, U, T, H, _p(q), _p(x), _p(attn), _p(q), None, _p(dq), _p(dx), _p(dS)),
    ]))
    assert rcs == [ERR_UNSUPPORTED] * 2 and launched == {}, (rcs, launched)


# ---- loss -----------------------------------------------------------------------------------------------------------
# Errors against float64 measured on an H100 80GB HBM3, largest over the cases below; the bounds keep about 4x.
LOSS_ROW_TOL = 6.0e-7   # measured 1.6e-7; in units of 1 + the row's largest |logit| (the loss is lse - x_y)
LOSS_GRAD_TOL = 1.5e-7  # measured 3.4e-8; in units of dloss[b] (1 + the row's largest |logit|): p = exp(x - lse) with
#                         lse rounded to fp32 is relatively off by |lse| eps


def loss_logits(rng, B, U, N):
    """[B*U][N]: utterance 0 normal, utterance 1 spread over +-80 and with one dominant class, utterance 2 normal"""
    x = rng.standard_normal((B, U, N)).astype(np.float32) * 3
    x[1, :2] = rng.uniform(-80, 80, (2, N)).astype(np.float32)
    x[1, 2] = rng.standard_normal(N).astype(np.float32)
    x[1, 2, N // 3] = 60.0
    x[1, 3] = rng.standard_normal(N).astype(np.float32)
    x[1, 3, 0] = 45.0
    return x.reshape(B * U, N)


@pytest.mark.parametrize("ls", [0.0, 0.1])
@pytest.mark.parametrize("N", [3, 31, 511, 512, 513, 65536])
def test_loss(N, ls):
    lib = _lib().lib
    B, U, pad = 3, 5, N - 1
    rng = np.random.default_rng(N * 7 + int(ls * 10))
    x = loss_logits(rng, B, U, N)
    y = rng.integers(0, N - 1, (B, U)).astype(np.int32)
    y[1, 2] = N // 3               # the dominant class is the target
    y[1, 3] = 1                    # the dominant class (0) is not
    y[0, 4] = pad
    y[2, 3:] = pad
    y[2, 1] = N                    # outside [0, N): that row's loss is NaN, its gradient 0
    y[2, 2] = -1
    dloss = np.array([0.5, -1.25, 2.0], np.float32)
    invalid = (y < 0) | (y >= N)
    pads = y == pad

    logits = torch.from_numpy(x).cuda()
    yd = torch.from_numpy(y).cuda()
    rowloss = torch.full((B * U,), 7.0, device="cuda")
    loss = torch.full((B,), 7.0, device="cuda")
    _ok(lib.w2l_seq2seq_loss(_s(), B, U, N, pad, _p(yd), _p(logits), ls, _p(torch.from_numpy(dloss).cuda()), 1, _p(rowloss), _p(loss),
                             None))
    rl = rowloss.cpu().numpy().reshape(B, U)
    grad = logits.cpu().numpy().reshape(B, U, N)

    # the per-utterance loss: a float32 sum of the row losses in row order
    want = np.zeros(B, np.float32)
    for b in range(B):
        for u in range(U):
            want[b] = np.float32(want[b] + rl[b, u])
    assert np.array_equal(loss.cpu().numpy(), want, equal_nan=True)

    x64 = torch.from_numpy(x).double().cuda().view(B, U, N)
    lp = torch.log_softmax(x64, -1)
    yl = torch.from_numpy(np.where(invalid, 0, y).astype(np.int64)).cuda()
    nll = -lp.gather(-1, yl[..., None])[..., 0]
    row = ((1 - ls) * nll - (ls / N) * lp.sum(-1)).cpu().numpy()
    g64 = lp.exp() - ls / N
    g64.scatter_add_(-1, yl[..., None], torch.full((B, U, 1), -(1 - ls), dtype=torch.float64, device="cuda"))
    g64 = (g64 * torch.from_numpy(dloss).double().cuda()[:, None, None]).cpu().numpy()

    assert np.isnan(rl[invalid]).all() and np.isnan(want[2])
    assert np.all(rl[pads] == 0) and np.all(grad[pads | invalid] == 0)
    ok = ~(pads | invalid)
    scale = 1 + np.abs(x.reshape(B, U, N)).max(-1)
    _within(f"loss.N{N}.ls{ls:g}.row", float((np.abs(rl - row) / scale)[ok].max()), LOSS_ROW_TOL)
    gerr = np.abs(grad - g64).max(-1) / np.abs(dloss)[:, None] / scale
    _within(f"loss.N{N}.ls{ls:g}.grad", float(gerr[ok].max()), LOSS_GRAD_TOL)

    # grad = 0 leaves the logits untouched and gives the same row losses; a flagged utterance is NaN throughout
    logits2 = torch.from_numpy(x).cuda()
    bad = torch.tensor([0, 1, 0], dtype=torch.int32, device="cuda")
    rowloss2, loss2 = torch.zeros_like(rowloss), torch.zeros_like(loss)
    _ok(lib.w2l_seq2seq_loss(_s(), B, U, N, pad, _p(yd), _p(logits2), ls, None, 0, _p(rowloss2), _p(loss2), _p(bad)))
    assert np.array_equal(logits2.cpu().numpy(), x)
    rl2 = rowloss2.cpu().numpy().reshape(B, U)
    assert np.isnan(rl2[1]).all() and np.isnan(loss2.cpu().numpy()[1])
    assert np.array_equal(rl2[[0, 2]], rl[[0, 2]], equal_nan=True)

    # scale_rows: d *= fp32(g[b] * fp32(1 / seed)), bit for bit
    gs = np.array([3.0, -0.7, 1.9], np.float32)
    seed = np.float32(1024.0 / 3.0)
    d = logits.clone()
    _ok(lib.w2l_seq2seq_scale_rows(_s(), B, U, N, _p(torch.from_numpy(gs).cuda()), float(seed), _p(d)))
    f = (gs * (np.float32(1) / seed)).astype(np.float32)
    assert np.array_equal(d.cpu().numpy().reshape(B, U, N), grad * f[:, None, None])


# ---- embedding gradient ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,U,H,N", [(40, 100, 96, 5000), (25, 120, 1024, 40000)])
def test_embed_bwd_bits(B, U, H, N):
    """dE[n] += s_n with s_n = 0 plus the rows of token n in row order (start token N: dstart), bit for bit"""
    lib = _lib().lib
    rng = np.random.default_rng(B * U + H)
    P = B * U
    tok = np.full((B, U), 7, np.int32)  # one token in most rows
    once = rng.random((B, U)) < 0.3
    tok[once] = rng.permutation(N)[:int(once.sum())]  # many tokens used once
    tok[:, 0] = N
    tok = tok.reshape(P)
    din = rng.standard_normal((P, H)).astype(np.float32)
    dE = rng.standard_normal((N, H)).astype(np.float32)
    dstart = rng.standard_normal(H).astype(np.float32)
    dE_d, dstart_d = torch.from_numpy(dE).cuda(), torch.from_numpy(dstart).cuda()
    _ok(lib.w2l_seq2seq_embed_bwd(_s(), B, U, H, N, _p(torch.from_numpy(tok).cuda()), _p(torch.from_numpy(din).cuda()), _p(dE_d),
                                  _p(dstart_d)))
    s = np.zeros((N + 1, H), np.float32)
    for k in range(P):
        s[tok[k]] += din[k]
    used = np.unique(tok)
    want = dE.copy()
    want[used[used < N]] += s[used[used < N]]
    assert (tok == 7).sum() > P // 2 and np.sum(np.bincount(tok) == 1) > P // 5
    assert np.array_equal(dE_d.cpu().numpy(), want)
    assert np.array_equal(dstart_d.cpu().numpy(), dstart + s[N])


# ---- greedy step ----------------------------------------------------------------------------------------------------
def first_max(row):
    """the kernel's argmax: NaN never wins, the first maximum does, token 0 if nothing beats -inf"""
    v = np.where(np.isnan(row), -np.inf, row)
    return int(np.argmax(v)) if np.any(v > -np.inf) else 0


def test_decode_step():
    lib = _lib().lib
    B, N, H, maxlen = 8, 65536, 32, 4
    eos, pad = N - 2, N - 1
    rng = np.random.default_rng(5)
    E = torch.from_numpy(rng.standard_normal((N, H)).astype(np.float32)).cuda()
    start = torch.from_numpy(rng.standard_normal(H).astype(np.float32)).cuda()
    inp = torch.zeros(B, H, device="cuda")
    tokens = torch.zeros(B, maxlen, dtype=torch.int32, device="cuda")
    length = torch.zeros(B, dtype=torch.int32, device="cuda")
    done = torch.full((B + 1,), 9, dtype=torch.int32, device="cuda")
    _ok(lib.w2l_seq2seq_decode_init(_s(), B, H, maxlen, pad, _p(start), _p(inp), _p(tokens), _p(length), _p(done)))
    assert torch.equal(inp, start.expand(B, H)) and torch.all(tokens == pad) and torch.all(length == maxlen)
    assert torch.all(done == 0)

    def logits_at(step):
        x = rng.integers(-40, 5, (B, N)).astype(np.float32)  # integer values: thousands of exact ties at the maximum
        x[1] = np.nan                                          # all NaN: token 0
        x[2, 77] = 9.0
        x[2, 77 + 256 * 5] = 9.0                               # two maxima in one thread's stride: the first wins
        x[3, :] = -np.inf                                      # nothing above -inf: token 0
        x[4, N - 1] = 9.0                                      # the last class
        x[5, ::3] = np.nan
        x[5, 3 * 1000 + 1] = 9.0                               # NaNs around the maximum
        x[6, eos] = 50.0 if step == 0 else -50.0               # eos: ends utterance 6 at step 0
        x[7, 300] = x[7, 300 + 256] = x[7, 31] = 7.0          # ties across threads: the lowest index
        return x

    want_tok = np.full((B, maxlen), pad, np.int32)
    want_len = np.full(B, maxlen, np.int32)
    want_in = inp.cpu().numpy().copy()
    fin = np.zeros(B, bool)
    En = E.cpu().numpy()
    for step in range(2):
        x = logits_at(step)
        _ok(lib.w2l_seq2seq_decode_step(_s(), B, N, H, step, eos, _p(torch.from_numpy(x).cuda()), _p(E), _p(inp), _p(tokens), maxlen,
                                        _p(length), _p(done)))
        for b in range(B):
            if fin[b]:
                continue
            t = first_max(x[b])
            if t == eos:
                fin[b], want_len[b] = True, step
            else:
                want_tok[b, step] = t
                want_in[b] = En[t]
        assert np.array_equal(tokens.cpu().numpy(), want_tok), step
        assert np.array_equal(length.cpu().numpy(), want_len), step
        assert np.array_equal(done.cpu().numpy(), np.append(fin.astype(np.int32), fin.sum())), step
        assert np.array_equal(inp.cpu().numpy(), want_in), step
    assert want_tok[2, 0] == 77 and want_tok[1, 0] == 0 and want_tok[3, 0] == 0 and want_len[6] == 0


# ---- beam search: the first step ------------------------------------------------------------------------------------
# score errors against float64, relative to max(1, |score|) (a score is x_c - lse, so its error is that of lse), measured
# on an H100 80GB HBM3
BEAM_SCORE_TOL = 5.0e-7  # measured 1.2e-7


def beam_logits(rng, B, K, N, eos):
    """[B*K][N] integer-valued rows for slot 0 (exact ties); the other slots are not live at step 0 and hold NaN"""
    x = np.full((B, K, N), np.nan, np.float32)
    lo = -30 if N > 100 else -3
    for b in range(B):
        x[b, 0] = rng.integers(lo, 1, N).astype(np.float32)
    if N > 100:
        x[:2, 0, eos] = -100.0                                  # eos out of reach
        x[1, 0, [40000, 123, N - 1, 7]] = [3.0, 3.0, 2.0, 2.0]  # a few keys above the ties, out of index order
        x[2, 0, eos] = 4.0                                      # eos first: a completion at rank 0
    else:
        x[2, 0, eos] = 1.0
    return x.reshape(B * K, N)


@pytest.mark.parametrize("K,N", [(1, 65536), (4, 65536), (16, 65536), (4, 5), (16, 29)])
def test_beam_first_step(K, N):
    """init, one step and finish over B utterances: the K live tokens and the completions, index for index against the
    float64 walk of tests/seq2seq_beam_reference.py, scores within BEAM_SCORE_TOL; N < 2K leaves each row fewer than 2K
    candidates"""
    lib = _lib().lib
    B, H, layers, maxlen = 3, 32, 1, 1
    eos, pad = N - 2, N - 1
    rng = np.random.default_rng(K * 100 + N)
    x = beam_logits(rng, B, K, N, eos)
    E = torch.from_numpy(rng.standard_normal((N, H)).astype(np.float32)).cuda()
    start = torch.from_numpy(rng.standard_normal(H).astype(np.float32)).cuda()
    nxt = torch.from_numpy(rng.standard_normal((layers, B * K, H)).astype(np.float32)).cuda()
    state = torch.zeros(layers, B * K, H, device="cuda")
    inp = torch.zeros(B * K, H, device="cuda")
    wsb = lib.w2l_seq2seq_beam_workspace_size(B, K, maxlen)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    _ok(lib.w2l_seq2seq_beam_init(_s(), B, K, H, maxlen, _p(start), _p(inp), _p(ws), wsb))
    assert torch.equal(inp, start.expand(B * K, H))
    _ok(lib.w2l_seq2seq_beam_step(_s(), B, K, N, H, layers, 0, maxlen, eos, _p(torch.from_numpy(x).cuda()), _p(E), _p(inp), _p(state),
                                  _p(nxt), _p(ws), wsb))
    toks = torch.zeros(B, K, maxlen, dtype=torch.int32, device="cuda")
    lens = torch.zeros(B, K, dtype=torch.int32, device="cuda")
    scores = torch.zeros(B, K, device="cuda")
    counts = torch.zeros(B, dtype=torch.int32, device="cuda")
    _ok(lib.w2l_seq2seq_beam_finish(_s(), B, K, maxlen, 1, pad, _p(ws), wsb, _p(toks), _p(lens), _p(scores), _p(counts)))
    toks, lens, scores, counts = toks.cpu().numpy(), lens.cpu().numpy(), scores.cpu().numpy(), counts.cpu().numpy()
    inp, state, En, nxt = inp.cpu().numpy(), state.cpu().numpy(), E.cpu().numpy(), nxt.cpu().numpy()
    stopped_count = int(ws[:4].view(torch.int32).item())

    start_np = start.cpu().numpy()
    xr = x.reshape(B, K, N)[:, 0].astype(np.float64)
    worst, stopped = 0.0, 0
    for b in range(B):
        lp = torch.log_softmax(torch.from_numpy(xr[b]), -1).numpy()
        live = []
        hyps, _ = beam(lambda st: (lp, lambda c: live.append(c)), None, K, 1, eos)
        order = sorted(range(N), key=lambda c: (-xr[b, c], c))
        # the live tokens are the best non-eos classes by (logit desc, class asc), as many as the walk reaches
        assert live == [c for c in order if c != eos][:K]
        # K completions (empty paths at step 0), the K-th above the best live score: the search of b stops there and its
        # inputs and states are left as they were
        stop = len(hyps) >= K and not hyps[0][1] and hyps[K - 1][0] > lp[live[0]]
        stopped += stop
        for slot, c in enumerate(live):
            assert np.array_equal(inp[b * K + slot], start_np if stop else En[c]), (b, slot)
            assert np.array_equal(state[0, b * K + slot], np.zeros(H, np.float32) if stop else nxt[0, b * K]), (b, slot)
        assert counts[b] == len(hyps), (b, counts[b], len(hyps))
        for k, (sc, path) in enumerate(hyps):
            assert lens[b, k] == len(path) and list(toks[b, k, :len(path)]) == path, (b, k)
            worst = max(worst, abs(scores[b, k] - sc) / max(1.0, abs(sc)))
        assert np.all(lens[b, len(hyps):] == 0) and np.all(scores[b, len(hyps):] == -np.inf)
        assert np.all(toks[b, len(hyps):] == pad)
    assert stopped_count == stopped
    _within(f"beam.K{K}.N{N}.score", float(worst), BEAM_SCORE_TOL)
