"""GPU checks of the converted GEMM kinds (F32X3, and TF32 with an MN-major operand): A is split in registers, B is
converted into its own ring.  Covers the TDS weight-gradient shapes, k-block counts that are not a multiple of either
ring's depth, an empty split-K slice, and bit-equality of the persistent and one-tile-per-CTA kernels."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# the weight gradients of the three TDS stages: dW[c][c] = dY^T X over the stage's frames
WGRAD_SHAPES = [(1440, 1440, 2400), (1120, 1120, 4800), (800, 800, 9600)]


def _operands(M, N, K, a_mn, b_mn, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn((K, M) if a_mn else (M, K), device="cuda", generator=g)
    B = torch.randn((K, N) if b_mn else (N, K), device="cuda", generator=g)
    return A, B


def _ratio(C, A, B, a_mn, b_mn, rel, C0=None):
    A64, B64 = (A.t() if a_mn else A).double(), (B.t() if b_mn else B).double()
    ref = A64 @ B64.t() + (C0.double() if C0 is not None else 0)
    bound = rel * (A64.abs() @ B64.abs().t()) + 1e-5
    return float(((C.double() - ref).abs() / bound).max())


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("M,N,K", WGRAD_SHAPES)
def test_f32x3_weight_gradient_shapes(M, N, K, accumulate):
    """fp32-accurate bound on the wgrad shapes (both operands MN-major, long K: split-K when the tiles under-fill the chip).
    The products are good to ~2^-21; the fp32 accumulation over K terms adds rounding that grows like sqrt(K), so the
    4e-6 bound of the K <= 1440 cases scales by sqrt(K / 1440)"""
    import wav2letter_b200 as w

    A, B = _operands(M, N, K, True, True, seed=K)
    C0 = torch.randn(M, N, device="cuda") * 10
    C = C0.clone()
    w.capi.gemm(A, B, "f32x3", True, True, out=C, accumulate=accumulate)
    torch.cuda.synchronize()
    ratio = _ratio(C, A, B, True, True, 4e-6 * (K / 1440) ** 0.5, C0 if accumulate else None)
    assert ratio <= 1.0, f"f32x3 wgrad M={M} N={N} K={K}: err/bound {ratio}"


@pytest.mark.parametrize("kind,rel", [("f32x3", 4e-6), ("tf32", 1.5e-3)])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("M,N,K", [(300, 260, 13 * 32), (132, 200, 7 * 32 - 4), (128, 128, 25 * 32)])
def test_converted_kinds_ring_wraparound_and_empty_slice(M, N, K, a_mn, b_mn, kind, rel):
    """13 and 7 k blocks are multiples of neither ring depth; 128 x 128 x 800 (one tile, 25 k blocks) splits K six ways
    in slices of 5, so the last slice is empty and writes zeros"""
    import wav2letter_b200 as w

    A, B = _operands(M, N, K, a_mn, b_mn, seed=M + K)
    C = w.capi.gemm(A, B, kind, a_mn, b_mn)
    torch.cuda.synchronize()
    ratio = _ratio(C, A, B, a_mn, b_mn, rel)
    assert ratio <= 1.0, f"{kind} M={M} N={N} K={K} a_mn={a_mn} b_mn={b_mn}: err/bound {ratio}"


@pytest.mark.parametrize("kind", ["tf32", "f32x3"])
@pytest.mark.parametrize("M,N,K,a_mn,b_mn", [(9600, 800, 800, False, False), (4800, 1120, 1120, False, True),
                                              (1120, 1120, 4800, True, True), (136, 72, 4000, True, False), (300, 10000, 1440, False, False)])
def test_converted_kinds_persistent_and_per_tile_are_bit_identical(M, N, K, a_mn, b_mn, kind):
    """both kernel variants walk the same tiles with the same k order and the same in-register split, so every result,
    split-K partial sums included, agrees to the last bit"""
    import wav2letter_b200 as w

    A, B = _operands(M, N, K, a_mn, b_mn, seed=M + N)
    bias = torch.randn(N, device="cuda")
    try:
        w.capi.gemm_set_variant(0)
        C0 = w.capi.gemm(A, B, kind, a_mn, b_mn, bias=bias, act=1)
        P0 = w.capi.gemm(A, B, kind, a_mn, b_mn)
        w.capi.gemm_set_variant(1)
        C1 = w.capi.gemm(A, B, kind, a_mn, b_mn, bias=bias, act=1)
        P1 = w.capi.gemm(A, B, kind, a_mn, b_mn)
    finally:
        w.capi.gemm_set_variant(1)
    torch.cuda.synchronize()
    assert torch.equal(C0, C1)
    assert torch.equal(P0, P1)
