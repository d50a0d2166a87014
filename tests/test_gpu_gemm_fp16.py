"""The FP16 operand kind of the wgmma GEMM (W2L_GEMM_FP16, csrc/gemm_wgmma.cu): the BF16 kernel template with fp16
operands.  fp16 operands are exact inputs here (the float64 reference is computed from the same fp16 values), so the only
error is fp32 accumulation, plus the fp16 rounding of C (2^-11 relative) when C is fp16.  Both majors of both operands,
both tile widths, split-K, the fp16-C and fp16-aux epilogues, the dynamic schedule (bit-identical to one tile per CTA)
and the fp16 casts."""
import pytest
import torch

pytestmark = pytest.mark.gpu

MAJORS = [(False, False), (False, True), (True, True), (True, False)]


def _operands(M, N, K, a_mn, b_mn, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn((K, M) if a_mn else (M, K), device="cuda", generator=g).half()
    B = torch.randn((K, N) if b_mn else (N, K), device="cuda", generator=g).half()
    return A, B


def _ref(A, B, a_mn, b_mn):
    A64, B64 = (A.t() if a_mn else A).double(), (B.t() if b_mn else B).double()
    return A64 @ B64.t(), A64.abs() @ B64.abs().t()


def _check(C, ref, mag, out16, what):
    bound = 2e-6 * mag + 1e-5 + (ref.abs() * 2.0 ** -11 if out16 else 0)
    ratio = float(((C.double() - ref).abs() / bound).max())
    assert ratio <= 1.0, f"{what}: err/bound {ratio}"


@pytest.mark.parametrize("out16", [False, True])
@pytest.mark.parametrize("a_mn,b_mn", MAJORS)
@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 384, 128), (200, 136, 104), (72, 56, 40), (4000, 800, 800),
                                   (1000, 2000, 1440), (1120, 1120, 4800)])
def test_gemm_fp16_kind(M, N, K, a_mn, b_mn, out16):
    import wav2letter_b200 as w

    A, B = _operands(M, N, K, a_mn, b_mn, seed=N + K)
    bias = torch.randn(N, device="cuda")
    C = w.capi.gemm(A, B, "fp16", a_mn, b_mn, bias=bias, act=1, out_bf16=out16)
    torch.cuda.synchronize()
    assert C.dtype == (torch.float16 if out16 else torch.float32)
    ref, mag = _ref(A, B, a_mn, b_mn)
    _check(C, (ref + bias.double()).clamp_min(0), mag, out16, f"fp16 M={M} N={N} K={K} a_mn={a_mn} b_mn={b_mn}")


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("a_mn,b_mn", MAJORS)
def test_gemm_fp16_tile_widths(a_mn, b_mn, bn):
    import wav2letter_b200 as w

    M, N, K = 520, 704, 392  # MN-major operands: rows of 16 bytes, 8 fp16
    A, B = _operands(M, N, K, a_mn, b_mn, seed=bn + 7)
    try:
        w.capi.gemm_set_tile(bn)
        C = w.capi.gemm(A, B, "fp16", a_mn, b_mn)
    finally:
        w.capi.gemm_set_tile(0)
    torch.cuda.synchronize()
    ref, mag = _ref(A, B, a_mn, b_mn)
    _check(C, ref, mag, False, f"fp16 BN={bn} a_mn={a_mn} b_mn={b_mn}")


@pytest.mark.parametrize("M,N,K,a_mn,b_mn", [(1120, 1120, 4800, True, True), (360, 360, 9600, True, True), (256, 200, 2056, False, False),
                                              (128, 128, 16 * 64, False, True)])
def test_gemm_fp16_split_k_accumulates_and_repeats(M, N, K, a_mn, b_mn):
    """weight-gradient shapes (few tiles, long K) are split along K; the slices are summed in a fixed order, so the
    result repeats bit for bit"""
    import wav2letter_b200 as w

    A, B = _operands(M, N, K, a_mn, b_mn, seed=M + K)
    C0 = torch.randn(M, N, device="cuda")
    outs = []
    for _ in range(3):
        C = C0.clone()
        w.capi.gemm(A, B, "fp16", a_mn, b_mn, out=C, accumulate=True)
        outs.append(C)
    torch.cuda.synchronize()
    ref, mag = _ref(A, B, a_mn, b_mn)
    _check(outs[0], ref + C0.double(), mag + C0.double().abs(), False, f"split-K M={M} N={N} K={K}")
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


def test_gemm_fp16_aux_mask_accumulate_and_view():
    import wav2letter_b200 as w

    # data-gradient shape with the activation mask read from an fp16 tensor and an fp32 accumulate
    A, B = _operands(300, 256, 160, False, True, seed=11)
    aux = torch.randn(300, 256, device="cuda").half()
    aux[::7] = 0
    for mode, keep in ((1, aux.double() > 0), (2, aux.double() != 0)):
        C0 = torch.randn(300, 256, device="cuda")
        C = C0.clone()
        w.capi.gemm(A, B, "fp16", False, True, out=C, accumulate=True, aux=aux, aux_mode=mode, aux_scale=1.25)
        ref = C0.double() + (A.double() @ B.double()) * keep * 1.25
        assert float((C.double() - ref).abs().max()) < 1e-3
    # the same with an fp16 C
    C16 = w.capi.gemm(A, B, "fp16", False, True, out_bf16=True, aux=aux, aux_mode=1, aux_scale=1.25)
    ref = (A.double() @ B.double()) * (aux.double() > 0) * 1.25
    assert C16.dtype == torch.float16
    assert float(((C16.double() - ref).abs() - ref.abs() * 2.0 ** -11).max()) < 1e-3
    # a bf16 aux is not an fp16 kind's aux
    with pytest.raises(TypeError):
        w.capi.gemm(A, B, "fp16", False, True, aux=aux.bfloat16(), aux_mode=1)
    # im2col view: rows of kw*Cin fp16 with row stride Cin
    T, Cin, Cout, kw = 300, 64, 96, 5
    x = torch.randn(T + kw - 1, Cin, device="cuda").half()
    wt = torch.randn(Cout, kw * Cin, device="cuda").half()
    y = torch.empty(T, Cout, device="cuda")
    w.capi.gemm(x, wt, "fp16", out=y, M=T, N=Cout, K=kw * Cin, lda=Cin, ldb=kw * Cin, allow_overlap=True)
    cols = torch.stack([x[t:t + kw].reshape(-1) for t in range(T)]).double()
    assert float((y.double() - cols @ wt.double().t()).abs().max()) < 2e-3


def test_gemm_fp16_dropout_mask_is_the_bf16_kinds():
    """the dropout mask hashes (seed, element index) only, so the fp16 and bf16 kinds drop the same elements"""
    import wav2letter_b200 as w

    A, B = _operands(384, 512, 256, False, False, seed=3)
    y16 = w.capi.gemm(A, B, "fp16", dropout_p=0.3, seed=1234)
    yb = w.capi.gemm(A.float().bfloat16(), B.float().bfloat16(), "bf16", dropout_p=0.3, seed=1234)
    torch.cuda.synchronize()
    assert torch.equal(y16 == 0, yb == 0)
    assert 0.25 < float((y16 == 0).float().mean()) < 0.35


# 2400 x 1440 x 1440: more than one wave of tiles, so the counter hands tiles out; 128 x 128 x 1600: one tile split along K
@pytest.mark.parametrize("a_mn,b_mn", MAJORS)
@pytest.mark.parametrize("M,N,K", [(2400, 1440, 1440), (304, 10000, 1440), (128, 128, 1600)])
def test_gemm_fp16_dynamic_schedule_matches_per_tile_kernel(M, N, K, a_mn, b_mn):
    import wav2letter_b200 as w

    A, B = _operands(M, N, K, a_mn, b_mn, seed=M + N + K)
    bias = torch.randn(N, device="cuda")

    def run():
        C = torch.full((M, N), float("nan"), device="cuda")
        P = torch.full((M, N), float("nan"), device="cuda")
        w.capi.gemm(A, B, "fp16", a_mn, b_mn, bias=bias, act=1, out=C)
        w.capi.gemm(A, B, "fp16", a_mn, b_mn, out=P)
        return C, P

    try:
        w.capi.gemm_set_variant(0)
        C0, P0 = run()
        w.capi.gemm_set_variant(1)
        C1, P1 = run()
    finally:
        w.capi.gemm_set_variant(1)
    torch.cuda.synchronize()
    assert not torch.isnan(P0).any()
    assert torch.equal(C0, C1)
    assert torch.equal(P0, P1)


def test_cast_fp16_matches_torch():
    import wav2letter_b200 as w

    x = torch.randn(1003, 37, device="cuda") * 5
    x[0, :4] = torch.tensor([7e4, -7e4, 65504.0, 1e-8])  # past the fp16 range: +-inf, as torch rounds
    assert torch.equal(w.capi.cast_fp16(x.reshape(-1)), x.reshape(-1).half())
    assert torch.equal(w.capi.cast_fp16(x.reshape(-1)[1:]), x.reshape(-1)[1:].half())  # unaligned: the scalar path
    y = w.capi.cast_fp16_rows(x, 40)
    assert torch.equal(y[:, :37], x.half()) and not y[:, 37:].any()
