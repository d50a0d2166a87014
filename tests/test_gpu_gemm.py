"""GPU parity of the wgmma/TMA GEMM (TF32 math, fp32 accumulate) against a float64 reference of
the same op.  Tolerance: TF32 keeps 10 mantissa bits per operand (TMA rounds on load), so each
product carries <= 2^-10 relative error: |C - ref| <= 1.5e-3 * (|A| |B|^T) element-wise."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def run(M, N, K, a_mn, b_mn, bias, act, seed=0):
    import wav2letter_b200 as w

    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn((K, M) if a_mn else (M, K), device="cuda", generator=g)
    B = torch.randn((K, N) if b_mn else (N, K), device="cuda", generator=g)
    bv = torch.randn(N, device="cuda", generator=g) if bias else None
    C = w.capi.gemm_tf32(A, B, bv, act, a_mn, b_mn)
    torch.cuda.synchronize()
    A64 = (A.t() if a_mn else A).double()
    B64 = (B.t() if b_mn else B).double()
    ref = A64 @ B64.t()
    bound = 1.5e-3 * (A64.abs() @ B64.abs().t()) + 1e-5
    if bias:
        ref = ref + bv.double()
    if act:
        ref = ref.clamp_min(0)
    err = (C.double() - ref).abs()
    ratio = float((err / bound).max())
    assert ratio <= 1.0, f"M={M} N={N} K={K} a_mn={a_mn} b_mn={b_mn}: err/bound {ratio}, max err {float(err.max())}"
    # and it must be a real TF32-accurate product, not garbage that happens to be small
    assert float(err.max()) < 0.05 * float(ref.abs().max()) + 1e-3


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True)])
@pytest.mark.parametrize("M,N,K", [(128, 128, 32), (128, 128, 256), (256, 384, 64), (200, 136, 100), (76, 52, 36),
                                   (4000, 800, 800), (1000, 2000, 1440)])
def test_gemm_majors_and_tails(M, N, K, a_mn, b_mn):
    run(M, N, K, a_mn, b_mn, bias=False, act=0, seed=M + N + K)


def test_gemm_bias_relu_epilogue():
    run(300, 1120, 1120, False, False, bias=True, act=1)
    run(130, 100, 64, False, False, bias=True, act=0)


def test_gemm_rejects_unaligned():
    import wav2letter_b200 as w

    A = torch.randn(8, 30, device="cuda")
    B = torch.randn(8, 30, device="cuda")
    with pytest.raises(w.W2LError):
        w.capi.gemm_tf32(A, B)


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("M,N,K,a_mn,b_mn", [(1120, 1120, 4800, True, True), (360, 360, 9600, True, True),
                                              (256, 200, 2052, False, False), (128, 128, 16 * 32, False, True)])
def test_gemm_split_k(M, N, K, a_mn, b_mn, accumulate):
    """few output tiles + long K (the weight-gradient shape): the k blocks are split into slices whose partial tiles are
    summed in slice order; same TF32 bound, plus the accumulate-onto-C semantics"""
    import wav2letter_b200 as w

    g = torch.Generator(device="cuda").manual_seed(K)
    A = torch.randn((K, M) if a_mn else (M, K), device="cuda", generator=g)
    B = torch.randn((K, N) if b_mn else (N, K), device="cuda", generator=g)
    C0 = torch.randn(M, N, device="cuda", generator=g) * 10
    C = C0.clone()
    w.capi.gemm_tf32_ex(A, B, C, a_mn=a_mn, b_mn=b_mn, accumulate=accumulate)
    torch.cuda.synchronize()
    A64 = (A.t() if a_mn else A).double()
    B64 = (B.t() if b_mn else B).double()
    ref = A64 @ B64.t() + (C0.double() if accumulate else 0)
    bound = 1.5e-3 * (A64.abs() @ B64.abs().t()) + 1e-4
    ratio = float(((C.double() - ref).abs() / bound).max())
    assert ratio <= 1.0, f"split-K M={M} N={N} K={K}: err/bound {ratio}"


@pytest.mark.parametrize("bn", [128, 160, 224, 256])
@pytest.mark.parametrize("M,N,K,a_mn,b_mn", [(1000, 800, 800, False, False), (700, 1120, 1120, False, True),
                                              (300, 1440, 1440, False, False), (1120, 1120, 2400, True, True),
                                              (200, 456, 100, False, True), (130, 10000, 64, False, False)])
def test_gemm_tile_widths(M, N, K, a_mn, b_mn, bn):
    """every tile width the host heuristic can pick (w2l_gemm_set_tile pins it), tails in M, N and K included"""
    import wav2letter_b200 as w

    w.capi.gemm_set_tile(bn)
    try:
        run(M, N, K, a_mn, b_mn, bias=not a_mn, act=0 if a_mn else 1, seed=bn + M)
    finally:
        w.capi.gemm_set_tile(0)


@pytest.mark.parametrize("T,Cin,Cout,kw", [(300, 40, 200, 13), (257, 100, 136, 5), (64, 244, 96, 21)])
def test_gemm_overlapping_rows_is_a_time_convolution(T, Cin, Cout, kw):
    """w2l_gemm_tf32_view: the im2col matrix of a stride-1 conv over [T][Cin] is rows of kw*Cin floats with row stride Cin
    (a zero-copy TMA view).  fwd (K-major view as A) and wgrad (MN-major view as B) against conv1d in float64."""
    import wav2letter_b200 as w

    g = torch.Generator(device="cuda").manual_seed(T)
    x = torch.randn(T, Cin, device="cuda", generator=g)
    wt = torch.randn(Cout, kw, Cin, device="cuda", generator=g) * 0.1   # arranged [co][dk*Cin + ci]
    bias = torch.randn(Cout, device="cuda", generator=g)
    Tout = T - kw + 1
    y = torch.empty(Tout, Cout, device="cuda")
    w.capi.gemm_tf32_view(x, Cin, wt.view(Cout, kw * Cin), kw * Cin, y, Tout, Cout, kw * Cin, bias=bias)
    ref = torch.nn.functional.conv1d(x.double().t().unsqueeze(0), wt.double().permute(0, 2, 1), bias.double())[0].t()
    assert float((y.double() - ref).abs().max()) < 3e-3 * float(ref.abs().max()) + 1e-3
    dy = torch.randn(Tout, Cout, device="cuda", generator=g)
    dw = torch.zeros(Cout, kw * Cin, device="cuda")
    w.capi.gemm_tf32_view(dy, Cout, x, Cin, dw, Cout, kw * Cin, Tout, a_mn=True, b_mn=True)
    cols = torch.stack([x[dk:dk + Tout] for dk in range(kw)], 1).reshape(Tout, kw * Cin).double()
    refw = dy.double().t() @ cols
    assert float((dw.double() - refw).abs().max()) < 3e-3 * float(refw.abs().max()) + 1e-3


@pytest.mark.parametrize("T,Cin,Cout,kw", [(52, 16, 40, 4), (300, 44, 200, 13)])
def test_gemm_view_data_gradient(T, Cin, Cout, kw):
    """data gradient of a stride-1 valid convolution: the view of dY padded with kw-1 zero rows in front (row t = frames
    t-(kw-1) .. t) times the flipped weights"""
    import wav2letter_b200 as w

    g = torch.Generator(device="cuda").manual_seed(T + kw)
    Tout = T - kw + 1
    dyp = torch.zeros(T + kw - 1, Cout, device="cuda")
    dyp[kw - 1:kw - 1 + Tout] = torch.randn(Tout, Cout, device="cuda", generator=g)
    wt = torch.randn(Cout, Cin, kw, device="cuda", generator=g) * 0.1   # [co][ci][dk]
    flip = wt.flip(2).permute(1, 2, 0).contiguous()                      # [ci][j][co], j = kw-1-dk
    dx = torch.empty(T, Cin, device="cuda")
    w.capi.gemm_tf32_view(dyp, Cout, flip.view(Cin, kw * Cout), kw * Cout, dx, T, Cin, kw * Cout)
    x64 = torch.zeros(1, Cin, T, dtype=torch.float64, device="cuda", requires_grad=True)
    y = torch.nn.functional.conv1d(x64, wt.double())
    y.backward(dyp[kw - 1:kw - 1 + Tout].double().t().unsqueeze(0))
    ref = x64.grad[0].t()
    assert float((dx.double() - ref).abs().max()) < 3e-3 * float(ref.abs().max()) + 1e-3


# ---- operand kinds: fp32-accurate 3xTF32 split and bf16 (csrc/gemm_wgmma.cu) ----------------------------------------
def _operands(M, N, K, a_mn, b_mn, seed, dtype=torch.float32):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn((K, M) if a_mn else (M, K), device="cuda", generator=g)
    B = torch.randn((K, N) if b_mn else (N, K), device="cuda", generator=g)
    return A.to(dtype), B.to(dtype)


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("M,N,K", [(128, 128, 32), (200, 136, 100), (76, 52, 36), (1000, 800, 1440), (360, 360, 9600)])
def test_gemm_f32x3_is_fp32_accurate(M, N, K, a_mn, b_mn):
    """error-compensated 3xTF32: |C - ref| <= 4e-6 * (|A| |B|^T) element-wise — 350x tighter than the TF32 bound, the
    accuracy class of an fp32 SGEMM (the reference's af::matmul -> cublasSgemm)"""
    import wav2letter_b200 as w

    A, B = _operands(M, N, K, a_mn, b_mn, seed=M + K)
    C = w.capi.gemm(A, B, "f32x3", a_mn, b_mn)
    torch.cuda.synchronize()
    A64, B64 = (A.t() if a_mn else A).double(), (B.t() if b_mn else B).double()
    ref = A64 @ B64.t()
    bound = 4e-6 * (A64.abs() @ B64.abs().t()) + 1e-6
    ratio = float(((C.double() - ref).abs() / bound).max())
    assert ratio <= 1.0, f"f32x3 M={M} N={N} K={K}: err/bound {ratio}"


def test_precision_switch_routes_fp32_entry_points():
    import wav2letter_b200 as w

    A, B = _operands(512, 320, 800, False, False, seed=3)
    ref = A.double() @ B.double().t()
    w.capi.set_precision("f32")
    try:
        C = w.capi.gemm_tf32(A, B)
    finally:
        w.capi.set_precision("tf32")
    C2 = w.capi.gemm_tf32(A, B)
    e1, e2 = float((C.double() - ref).abs().max()), float((C2.double() - ref).abs().max())
    assert e1 < 2e-4 and e2 > 10 * e1, (e1, e2)  # fp32-accurate vs TF32 rounding


@pytest.mark.parametrize("out_bf16", [False, True])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 384, 128), (200, 136, 104), (72, 56, 40), (4000, 800, 800),
                                   (1000, 2000, 1440), (1120, 1120, 4800)])
def test_gemm_bf16_kind(M, N, K, a_mn, b_mn, out_bf16):
    """bf16 operands are exact inputs here (the reference is computed from the same bf16 values), so the only error is
    fp32 accumulation (+ the bf16 rounding of C when out_bf16)"""
    import wav2letter_b200 as w

    A, B = _operands(M, N, K, a_mn, b_mn, seed=N + K, dtype=torch.bfloat16)
    bias = torch.randn(N, device="cuda")
    C = w.capi.gemm(A, B, "bf16", a_mn, b_mn, bias=bias, act=1, out_bf16=out_bf16)
    torch.cuda.synchronize()
    assert C.dtype == (torch.bfloat16 if out_bf16 else torch.float32)
    A64, B64 = (A.t() if a_mn else A).double(), (B.t() if b_mn else B).double()
    ref = (A64 @ B64.t() + bias.double()).clamp_min(0)
    bound = 2e-6 * (A64.abs() @ B64.abs().t()) + 1e-5 + (ref.abs() * 2.0 ** -8 if out_bf16 else 0)
    ratio = float(((C.double() - ref).abs() / bound).max())
    assert ratio <= 1.0, f"bf16 M={M} N={N} K={K} a_mn={a_mn} b_mn={b_mn}: err/bound {ratio}"


def test_gemm_bf16_mask_accumulate_and_view():
    import wav2letter_b200 as w

    # data-gradient shape with the activation mask read from a bf16 tensor and an fp32 accumulate
    A, B = _operands(300, 256, 160, False, True, seed=11, dtype=torch.bfloat16)
    aux = torch.randn(300, 256, device="cuda").to(torch.bfloat16)
    C0 = torch.randn(300, 256, device="cuda")
    C = C0.clone()
    w.capi.gemm(A, B, "bf16", False, True, out=C, accumulate=True, aux=aux, aux_mode=1, aux_scale=1.25)
    ref = C0.double() + (A.double() @ B.double()) * (aux.double() > 0) * 1.25
    assert float((C.double() - ref).abs().max()) < 1e-3
    # im2col view: rows of kw*Cin bf16 with row stride Cin
    T, Cin, Cout, kw = 300, 64, 96, 5
    x = torch.randn(T + kw - 1, Cin, device="cuda").to(torch.bfloat16)
    wt = torch.randn(Cout, kw * Cin, device="cuda").to(torch.bfloat16)
    y = torch.empty(T, Cout, device="cuda")
    w.capi.gemm(x, wt, "bf16", out=y, M=T, N=Cout, K=kw * Cin, lda=Cin, ldb=kw * Cin, allow_overlap=True)
    cols = torch.stack([x[t:t + kw].reshape(-1) for t in range(T)]).double()
    assert float((y.double() - cols @ wt.double().t()).abs().max()) < 2e-3


def test_cast_bf16_matches_torch():
    import wav2letter_b200 as w

    x = torch.randn(1003, 37, device="cuda") * 5
    assert torch.equal(w.capi.cast_bf16(x.reshape(-1)), x.reshape(-1).to(torch.bfloat16))


@pytest.mark.parametrize("kind", ["tf32", "f32x3", "bf16"])
@pytest.mark.parametrize("M,N,K,a_mn,b_mn", [(9600, 800, 800, False, False), (4800, 1120, 1120, False, True), (1120, 1120, 4800, True, True),
                                              (300, 10000, 1440, False, False), (136, 72, 4000, True, False), (128, 128, 64, False, False)])
def test_gemm_persistent_and_per_tile_kernels_agree(M, N, K, a_mn, b_mn, kind):
    """the persistent kernel (one CTA per SM walking the tiles) against the one-tile-per-CTA kernel: same tile
    shape, k order and split-K slice order, so results agree to the last bit"""
    import wav2letter_b200 as w

    A, B = _operands(M, N, K, a_mn, b_mn, seed=M + N, dtype=torch.bfloat16 if kind == "bf16" else torch.float32)
    bias = torch.randn(N, device="cuda")
    try:
        w.capi.gemm_set_tile(128)
        w.capi.gemm_set_variant(0)
        C0 = w.capi.gemm(A, B, kind, a_mn, b_mn, bias=bias, act=1)
        P0 = w.capi.gemm(A, B, kind, a_mn, b_mn)  # plain: may split K
        w.capi.gemm_set_variant(1)
        C1 = w.capi.gemm(A, B, kind, a_mn, b_mn, bias=bias, act=1)
        P1 = w.capi.gemm(A, B, kind, a_mn, b_mn)
    finally:
        w.capi.gemm_set_variant(1)
        w.capi.gemm_set_tile(0)
    torch.cuda.synchronize()
    if kind == "f32x3":  # the two kernels round the hi / lo split differently (cvt.rna vs integer round-to-nearest)
        assert float((C0 - C1).abs().max()) <= 2e-5 * float(C0.abs().max())
    else:
        assert torch.equal(C0, C1)
    assert float((P0 - P1).abs().max()) <= 1e-4 * float(P0.abs().max()) + 1e-6
    ref = (A.t() if a_mn else A).double() @ (B.t() if b_mn else B).double().t()
    tol = {"tf32": 3e-3, "f32x3": 2e-5, "bf16": 2e-5}[kind]
    assert float((P1.double() - ref).abs().max()) <= tol * float(ref.abs().max()) * (K ** 0.5) / 8 + 1e-4


@pytest.mark.parametrize("kind", ["tf32", "f32x3", "bf16"])
def test_gemm_split_k_is_run_to_run_identical(kind):
    """split-K partial tiles are summed in slice order, so repeating a weight-gradient-shaped GEMM gives the same bits"""
    import wav2letter_b200 as w

    A, B = _operands(360, 360, 9600, True, True, seed=5, dtype=torch.bfloat16 if kind == "bf16" else torch.float32)
    C0 = torch.randn(360, 360, device="cuda")
    outs = []
    for _ in range(3):
        C = C0.clone()
        w.capi.gemm(A, B, kind, True, True, out=C, accumulate=True)
        outs.append(C)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
