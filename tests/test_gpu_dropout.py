"""Every dropout site bit-exact against its NumPy model (tests/dropout_reference.py), the forward-to-backward mask
handoff as fl_compat wires it, and SpecAugment's band masking against NumPy.

Pre-dropout values are made exact on every arithmetic path: activations are integers in [-8, 8], weights in {-1, 0, 1},
biases integers, so TF32, 3xTF32 and bf16 products and their fp32 sums carry no rounding, and the expected output
`pre * scale (+ add)` is computed in NumPy float32 and compared with torch.equal.  Where a residual `add` follows the
dropout, p is 0.5 or 0.75 (scale 2 or 4, so pre * scale is exact and a fused multiply-add rounds like the separate
operations).

The backward passes never regenerate a mask: they read it back from the stored activation, and an exactly-zero stored
value reads as dropped.  That is the true gradient whenever a ReLU precedes the dropout (a zero ReLU output has zero
gradient either way); for dropout alone it zeroes the gradient of kept elements whose value is exactly 0."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dropout_reference as R

pytestmark = pytest.mark.gpu

P_ODD = 0.590432749713  # the conv_glu LibriSpeech arch's largest dropout: scale 1/(1-p) is not a short binary fraction


def capi():
    from wav2letter_b200 import capi as c

    return c


def ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, shape, generator=g, device="cuda").float()


def ref_conv64(x, wt, bias, stride, pad_left, Tout):
    """x [B,T,Cin,W], wt [Cout,Cin,K] -> [B,Tout,Cout,W] in float64"""
    K = wt.shape[2]
    xin = x.double().permute(0, 2, 1, 3)
    pad_right = max(0, (Tout - 1) * stride + K - x.shape[1] - pad_left)
    xin = F.pad(xin, (0, 0, pad_left, pad_right))
    y = F.conv2d(xin, wt.double().unsqueeze(-1), None if bias is None else bias.double(), stride=(stride, 1))
    return y[:, :, :Tout].permute(0, 2, 1, 3).contiguous()


def model_scale(fn, seed, shape, p, **kw):
    e = np.arange(int(np.prod(shape)), dtype=np.uint64)
    return torch.from_numpy(fn(seed, e, p, **kw).reshape(shape)).cuda()


def kernels_run(fn):
    names = capi().trace(fn)
    return set(names)


# ---------------------------------------------------------------------------------------------------------------------
# time convolution forward: SIMT (W % 8 != 0), mma.sync TF32 and 3xTF32 (W2L_PRECISION_F32)
# ---------------------------------------------------------------------------------------------------------------------
CONV_KERNEL = {"simt": "conv_time_fwd_kernel", "mma": "conv_mma_fwd_kernel", "x3": "conv_mma_fwd_kernel"}
CONV_CASES = [  # path, B, T, Cin, Cout, K, stride, W
    ("simt", 2, 23, 5, 7, 3, 1, 20), ("simt", 3, 30, 4, 13, 5, 2, 36), ("simt", 2, 19, 6, 27, 3, 1, 76),
    ("mma", 2, 21, 5, 7, 3, 1, 8), ("mma", 2, 26, 6, 13, 5, 2, 16), ("mma", 3, 19, 4, 9, 3, 1, 24), ("mma", 2, 20, 5, 27, 3, 1, 32),
    ("mma", 2, 33, 7, 17, 5, 2, 40), ("mma", 2, 30, 10, 10, 5, 1, 80),
    ("x3", 2, 21, 5, 13, 3, 1, 24), ("x3", 2, 30, 6, 27, 5, 2, 80),
    ("mma", 2, 35, 9, 18, 5, 1, 8), ("mma", 2, 35, 9, 18, 5, 2, 24), ("mma", 2, 35, 9, 18, 5, 1, 40), ("mma", 2, 35, 9, 18, 5, 2, 80),
    ("x3", 2, 35, 9, 18, 5, 1, 8), ("x3", 2, 35, 9, 18, 5, 2, 24), ("x3", 2, 35, 9, 18, 5, 1, 40), ("x3", 2, 35, 9, 18, 5, 2, 80),
]


def run_conv(path, *args, **kw):
    c = capi()
    try:
        c.set_precision("f32" if path == "x3" else "tf32")
        out = {}
        ran = kernels_run(lambda: out.setdefault("y", c.conv_time_fwd(*args, **kw)))
        return out["y"], ran
    finally:
        c.set_precision("tf32")


@pytest.mark.parametrize("path,B,T,Cin,Cout,K,stride,W", CONV_CASES)
def test_conv_time_fwd_dropout_matches_model(path, B, T, Cin, Cout, K, stride, W):
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + T * 10 + W)
    x = ints((B, T, Cin, W), -8, 8, g)
    wt = ints((Cout, Cin, K), -1, 1, g)
    bias = ints((Cout,), -3, 3, g)
    pl = K // 2
    Tout = (T + 2 * pl - K) // stride + 1
    pre = ref_conv64(x, wt, bias, stride, pl, Tout).float()  # exact integers
    add = ints((B, Tout, Cout, W), -8, 8, g)
    fn, kw = {"simt": (R.simt_scale, {}), "mma": (R.conv_mma_scale, dict(W=W)), "x3": (R.conv_mma_scale, dict(W=W))}[path]
    seed = R.host_seed(W + Cout)
    for act, p, residual in ((0, 0.2, False), (1, P_ODD, False), (0, 0.5, True), (1, 0.75, True)):
        y, ran = run_conv(path, x, wt, bias, Tout, stride, pl, act=act, dropout_p=p, seed=seed, add=add if residual else None)
        assert CONV_KERNEL[path] in ran, (path, ran)
        a = pre.clamp_min(0) if act else pre
        s = model_scale(fn, seed, y.shape, p, **kw)
        want = a * s + (add if residual else 0)
        assert torch.equal(y, want), (path, act, p, residual, int((y != want).sum()))
        y2, _ = run_conv(path, x, wt, bias, Tout, stride, pl, act=act, dropout_p=p, seed=seed, add=add if residual else None)
        assert torch.equal(y, y2)
    y3, _ = run_conv(path, x, wt, bias, Tout, stride, pl, act=1, dropout_p=0.75, seed=seed + 1, add=add)
    assert not torch.equal(y, y3)


# ---------------------------------------------------------------------------------------------------------------------
# GEMM epilogue
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["tf32", "f32x3", "bf16"])
@pytest.mark.parametrize("c_bf16", [False, True])
def test_gemm_epilogue_dropout_matches_model(kind, c_bf16):
    c = capi()
    g = torch.Generator(device="cuda").manual_seed(17)
    M, N, K = 300, 356, 72  # M: a 44-row tail; N % 4 == 0 but no tile width divides it
    A, Bm, bias = ints((M, K), -8, 8, g), ints((N, K), -1, 1, g), ints((N,), -4, 4, g)
    pre = (A.double() @ Bm.double().t() + bias.double()).float()
    if kind == "bf16":
        A, Bm = A.bfloat16(), Bm.bfloat16()
    seed = R.host_seed(40)
    outs = []
    try:
        for variant in (0, 1):
            for bn in (128, 160, 224, 256):
                c.gemm_set_variant(variant)
                c.gemm_set_tile(bn)
                for act, p in ((1, 0.2), (0, P_ODD)):
                    y = c.gemm(A, Bm, kind=kind, bias=bias, act=act, out_bf16=c_bf16, dropout_p=p, seed=seed)
                    want = (pre.clamp_min(0) if act else pre) * model_scale(R.gemm_scale, seed, (M, N), p)
                    if c_bf16:
                        want = want.bfloat16()
                    assert torch.equal(y, want), (kind, c_bf16, variant, bn, act, int((y != want).sum()))
                    outs.append(y)
                y2 = c.gemm(A, Bm, kind=kind, bias=bias, act=0, out_bf16=c_bf16, dropout_p=P_ODD, seed=seed + 1)
                assert not torch.equal(y2, outs[-1])
    finally:
        c.gemm_set_variant(1)
        c.gemm_set_tile(0)


@pytest.mark.parametrize("precision", ["tf32", "f32"])
def test_gemm_tf32_ex_dropout_matches_model(precision):
    c = capi()
    g = torch.Generator(device="cuda").manual_seed(23)
    M, N, K = 517, 132, 40
    A, Bm, bias = ints((M, K), -8, 8, g), ints((N, K), -1, 1, g), ints((N,), -4, 4, g)
    pre = (A.double() @ Bm.double().t() + bias.double()).float().clamp_min(0)
    seed = R.host_seed(41)
    out = torch.empty((M, N), device="cuda")
    try:
        c.set_precision(precision)
        c.gemm_tf32_ex(A, Bm, out, bias=bias, act=1, dropout_p=0.25, seed=seed)
    finally:
        c.set_precision("tf32")
    assert torch.equal(out, pre * model_scale(R.gemm_scale, seed, (M, N), 0.25))


# ---------------------------------------------------------------------------------------------------------------------
# GLU forward / backward: float4 path (half % 4 == 0, 16-byte aligned) and scalar path
# ---------------------------------------------------------------------------------------------------------------------
def glu_call(x, dy, H, p, seed, offset):
    """w2l_glu_fwd / bwd on copies of x, dy placed `offset` floats into their buffers (offset 1 forces the scalar path)"""
    c = capi()
    R_ = x.shape[0]

    def place(t):
        buf = torch.zeros(t.numel() + 4, device="cuda")
        v = buf[offset:offset + t.numel()].view(t.shape)
        v.copy_(t)
        return v

    xs, dys = place(x), place(dy)
    y = place(torch.zeros(R_, H, device="cuda"))
    dx = place(torch.zeros_like(x))
    c._check(c.lib.w2l_glu_fwd(c._stream(), R_, H, c._ptr(xs), c._ptr(y), p, seed))
    c._check(c.lib.w2l_glu_bwd(c._stream(), R_, H, c._ptr(xs), c._ptr(dys), c._ptr(dx), p, seed))
    return y.clone(), dx.clone()


@pytest.mark.parametrize("rows,H", [(1000, 256), (700, 260), (900, 122), (333, 7)])
def test_glu_dropout_fwd_bwd_match_model(rows, H):
    g = torch.Generator(device="cuda").manual_seed(rows + H)
    x = torch.randn(rows, 2 * H, device="cuda", generator=g)
    x[:, :H] += torch.sign(x[:, :H]) * 0.05  # a != 0: the output is zero exactly where the mask drops
    dy = torch.randn(rows, H, device="cuda", generator=g)
    seed, p = R.host_seed(50 + H), 0.25
    fn = R.glu_vec_scale if H % 4 == 0 else R.simt_scale
    kw = dict(H=H) if H % 4 == 0 else {}
    s = model_scale(fn, seed, (rows, H), p, **kw).double()
    y, dx = glu_call(x, dy, H, p, seed, 0)
    a, b = x[:, :H].double(), x[:, H:].double()
    sg = torch.sigmoid(b)
    yr = a * sg * s
    assert torch.equal(y == 0, s == 0)
    assert float((y.double() - yr).abs().max() / yr.abs().max()) < 1e-6
    d = dy.double() * s
    dxr = torch.cat([d * sg, d * a * sg * (1 - sg)], dim=1)
    assert torch.equal(dx[:, :H] == 0, s == 0)  # backward applies the forward's mask
    assert float((dx.double() - dxr).abs().max() / dxr.abs().max()) < 1e-6
    if H % 4 == 0:  # the scalar path (pointers off 16-byte alignment) draws the same bits
        y1, dx1 = glu_call(x, dy, H, p, seed, 1)
        assert torch.equal(y1, y) and torch.equal(dx1, dx)
    y2, dx2 = glu_call(x, dy, H, p, seed, 0)
    assert torch.equal(y2, y) and torch.equal(dx2, dx)
    y3, _ = glu_call(x, dy, H, p, seed + 1, 0)
    assert not torch.equal(y3 == 0, y == 0)


# ---------------------------------------------------------------------------------------------------------------------
# standalone ReLU / Dropout and their backward mask
# ---------------------------------------------------------------------------------------------------------------------
def act_fwd(x, relu, p, seed):
    c = capi()
    y = torch.empty_like(x)
    c._check(c.lib.w2l_act_fwd(c._stream(), x.numel(), c._ptr(x), relu, p, seed, c._ptr(y)))
    return y


def mask_mul(gr, ref, mode, scale):
    c = capi()
    out = torch.empty_like(gr)
    c._check(c.lib.w2l_mask_mul(c._stream(), gr.numel(), c._ptr(gr), c._ptr(ref), mode, scale, c._ptr(out)))
    return out


@pytest.mark.parametrize("relu", [0, 1])
@pytest.mark.parametrize("p", [0.1, P_ODD])
def test_act_fwd_dropout_matches_model(relu, p):
    g = torch.Generator(device="cuda").manual_seed(31 + relu)
    n = 1_000_003
    x = torch.randn(n, device="cuda", generator=g)
    x[::97] = 0.0
    seed = R.host_seed(60 + relu)
    y = act_fwd(x, relu, p, seed)
    s = model_scale(R.simt_scale, seed, (n,), p)
    assert torch.equal(y, (x.clamp_min(0) if relu else x) * s)
    assert torch.equal(act_fwd(x, relu, p, seed), y)
    assert not torch.equal(act_fwd(x, relu, p, seed + 1), y)


@pytest.mark.parametrize("mode", [1, 2])
def test_mask_mul(mode):
    g = torch.Generator(device="cuda").manual_seed(37)
    n = 777_777
    ref = torch.randn(n, device="cuda", generator=g)
    ref[::5] = 0.0
    ref[1::11] = -0.0
    gr = torch.randn(n, device="cuda", generator=g)
    scale = float(R.keep_scale(P_ODD))
    out = mask_mul(gr, ref, mode, scale)
    keep = ref > 0 if mode == 1 else ref != 0
    assert torch.equal(out, torch.where(keep, torch.tensor(np.float32(scale), device="cuda"), 0.0) * gr)


# ---------------------------------------------------------------------------------------------------------------------
# forward-to-backward handoff (fl_compat: Conv2D with fused ReLU + dropout, Linear with dropout in the GEMM epilogue and
# the mask in the consumer's data-gradient epilogue, standalone ReLU -> Dropout)
# ---------------------------------------------------------------------------------------------------------------------
def test_conv_relu_dropout_backward_uses_the_forward_mask():
    c = capi()
    g = torch.Generator(device="cuda").manual_seed(41)
    B, T, Cin, Cout, K, W, p = 2, 30, 6, 10, 5, 80, 0.5
    x, wt, bias = ints((B, T, Cin, W), -8, 8, g), ints((Cout, Cin, K), -1, 1, g), ints((Cout,), -2, 2, g)
    seed = R.host_seed(70)
    y = c.conv_time_fwd(x, wt, bias, T, 1, 2, act=1, dropout_p=p, seed=seed)
    dy = ints(y.shape, -8, 8, g)
    keep = float(R.keep_scale(p))
    dpre = mask_mul(dy, y, 1, keep)  # Conv2D's backward: the mask read from the stored output (ReLU zeros included)
    x64, w64, b64 = x.double().requires_grad_(True), wt.double().requires_grad_(True), bias.double().requires_grad_(True)
    pre = ref_conv64(x64, w64, b64, 1, 2, T)
    assert bool((pre == 0).any()) and bool((y == 0).any())
    out = F.relu(pre) * model_scale(R.simt_scale, seed, y.shape, p).double()
    out.backward(dy.double())
    dpre_ref = dy.double() * (pre.detach() > 0) * model_scale(R.simt_scale, seed, y.shape, p).double()
    assert torch.equal(dpre.double(), dpre_ref)
    dx = c.conv_time_dgrad(dpre, wt, T, 1, 2)
    dwt, dbias = c.conv_time_wgrad(x, dpre, K, 1, 2)
    assert torch.equal(dx.double(), x64.grad)  # integer gradients: exact on every path
    assert torch.equal(dwt.double(), w64.grad) and torch.equal(dbias.double(), b64.grad)


@pytest.mark.parametrize("relu", [1, 0])
def test_linear_dropout_backward_through_aux_mask(relu):
    """h = dropout(act(x W1^T + b1)) in the GEMM epilogue; the consumer's data gradient dh = (dz W2) * mask(h) * keep with
    the mask read from h (aux_mode 1: h > 0 after a ReLU, 2: h != 0)"""
    c = capi()
    g = torch.Generator(device="cuda").manual_seed(43 + relu)
    M, nin, nh, nout, p = 260, 48, 132, 36, 0.5
    x, w1, b1 = ints((M, nin), -8, 8, g), ints((nh, nin), -1, 1, g), ints((nh,), -3, 3, g)
    w2 = ints((nout, nh), -1, 1, g)  # [out][in]: the data gradient reads it MN-major
    seed = R.host_seed(80 + relu)
    h = c.gemm(x, w1, bias=b1, act=relu, dropout_p=p, seed=seed)
    pre = x.double() @ w1.double().t() + b1.double()
    s = model_scale(R.gemm_scale, seed, (M, nh), p).double()
    assert torch.equal(h.double(), (pre.clamp_min(0) if relu else pre) * s)
    assert bool((pre == 0).any())  # exact zeros in the stored activation
    dz = ints((M, nout), -8, 8, g)
    dh = c.gemm(dz, w2, b_mn=True, aux=h, aux_mode=1 if relu else 2, aux_scale=float(R.keep_scale(p)))
    d = dz.double() @ w2.double()
    if relu:
        want = d * s * (pre > 0)  # the true gradient of dropout(relu(.))
    else:
        want = d * s * (pre != 0)  # the pinned rule: a kept exact zero reads as dropped
        assert bool(((pre == 0) & (s != 0)).any())
    assert torch.equal(dh.double(), want)


def test_standalone_relu_then_dropout_backward():
    g = torch.Generator(device="cuda").manual_seed(47)
    n, p = 300_001, 0.2
    x = torch.randn(n, device="cuda", generator=g)
    x[::13] = 0.0
    seed = R.host_seed(90)
    r = act_fwd(x, 1, 0.0, 0)
    y = act_fwd(r, 0, p, seed)
    gy = torch.randn(n, device="cuda", generator=g)
    keep = float(R.keep_scale(p))
    gr = mask_mul(gy, y, 2, keep)  # Dropout's backward
    gx = mask_mul(gr, r, 1, 1.0)   # ReLU's backward
    s = model_scale(R.simt_scale, seed, (n,), p)
    assert torch.equal(y, x.clamp_min(0) * s)
    assert torch.equal(gx, torch.where(x > 0, gy * s, 0.0))


# ---------------------------------------------------------------------------------------------------------------------
# SpecAugment band masking
# ---------------------------------------------------------------------------------------------------------------------
def mask_bands(x, fb, tb, value):
    c = capi()
    B, T, C, W = x.shape
    y = torch.empty_like(x)

    def arr(vals):
        a = (ctypes.c_int * max(1, len(vals)))(*vals)
        return a, ctypes.cast(a, ctypes.c_void_p)

    keep = [arr([f for f, _ in fb]), arr([f for _, f in fb]), arr([t for t, _ in tb]), arr([t for _, t in tb])]
    rc = c.lib.w2l_mask_bands(c._stream(), B, T, C, W, c._ptr(x), c._ptr(y), len(fb), keep[0][1], keep[1][1], len(tb), keep[2][1],
                              keep[3][1], value)
    return rc, y


BANDS = [
    ([], [], 0.0),
    ([(0, 3)], [], 0.0),
    ([], [(0, 1)], -2.5),
    ([(5, 9), (7, 12), (26, 29)], [(3, 10), (35, 37)], -2.5),
    ([(0, 29)], [(0, 37)], 1.75),
    ([(1, 2), (4, 4), (3, 8), (28, 29), (0, 1), (10, 20), (12, 15), (20, 21)],
     [(0, 2), (2, 5), (36, 37), (10, 10), (11, 30), (12, 13), (30, 31), (31, 36)], 3.0),
]


@pytest.mark.parametrize("fb,tb,value", BANDS)
def test_mask_bands_matches_numpy(fb, tb, value):
    g = torch.Generator(device="cuda").manual_seed(53)
    B, T, C, W = 3, 37, 5, 29
    x = torch.randn(B, T, C, W, device="cuda", generator=g)
    rc, y = mask_bands(x, fb, tb, value)
    assert rc == 0
    want = x.cpu().numpy().copy()
    for f0, f1 in fb:
        want[:, :, :, f0:f1] = value
    for t0, t1 in tb:
        want[:, t0:t1] = value
    assert np.array_equal(y.cpu().numpy(), want)


def test_mask_bands_rejects_more_than_eight_bands():
    x = torch.zeros(1, 4, 2, 10, device="cuda")
    rc, _ = mask_bands(x, [(0, 1)] * 9, [], 0.0)
    assert rc == 4  # W2L_ERR_UNSUPPORTED
    rc, _ = mask_bands(x, [], [(0, 1)] * 9, 0.0)
    assert rc == 4
