"""F32X3 with B pre-split into tf32 hi / lo planes (w2l_split_tf32 + kind f32x3_split_b).

The split must round exactly as the F32X3 kernel's in-tile conversion (hi = tf32(x), lo = tf32(x - hi), round to nearest
with ties away from zero on the bit pattern), and the split-B kernel issues the same MMAs in the same order, so its
results must equal plain F32X3 on the unsplit B bit for bit: at the train step's shapes, on ragged edges, with every
epilogue and under every schedule."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def rn_tf32(u):
    return ((u.astype(np.uint64) + 0x1000) & 0xFFFFE000).astype(np.uint32)


def split_model(x, transpose, cols_padded):
    """NumPy model of w2l_split_tf32: [2][R][cols_padded] float32"""
    src = x.T if transpose else x
    hi = rn_tf32(np.ascontiguousarray(src).view(np.uint32))
    lo = rn_tf32((src - hi.view(np.float32)).astype(np.float32).view(np.uint32))
    out = np.zeros((2, src.shape[0], cols_padded), np.uint32)
    out[0, :, : src.shape[1]] = hi
    out[1, :, : src.shape[1]] = lo
    return out


@pytest.mark.parametrize("rows,cols,transpose,cols_padded", [
    (800, 800, False, 800), (1440, 10000, False, 10000), (1440, 10000, True, 1440), (1120, 1120, True, 1120),
    (1000, 375, False, 376),  # padded K (a WSJ-style Linear)
    (375, 1000, True, 380),  # transposed, padded K, rows and columns not multiples of the 32 x 32 tile
    (37, 45, True, 64), (45, 37, False, 40),
])
def test_split_planes_bit_equal_to_model(rows, cols, transpose, cols_padded):
    import wav2letter_b200 as w

    g = np.random.default_rng(rows * 7 + cols)
    x = (g.standard_normal((rows, cols)) * np.exp2(g.integers(-20, 20, (rows, cols)))).astype(np.float32)
    # rounding ties (the 13 dropped bits exactly 0x1000) and neighbours, both signs
    u = x.reshape(-1).view(np.uint32)
    u[:64] = (u[:64] & 0xFFFFE000) | np.array([0x1000, 0x0FFF, 0x1001, 0x1FFF] * 16, np.uint32)
    got = w.capi.split_tf32(torch.from_numpy(x).cuda(), transpose=transpose, cols_padded=cols_padded)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(got.cpu().numpy().view(np.uint32), split_model(x, transpose, cols_padded))


def test_split_of_a_row_strided_view():
    import wav2letter_b200 as w

    big = torch.randn(300, 260, device="cuda")
    x = big[:, :250]  # row stride 260
    for transpose in (False, True):
        got = w.capi.split_tf32(x, transpose=transpose)
        want = split_model(x.contiguous().cpu().numpy(), transpose, got.shape[2])
        np.testing.assert_array_equal(got.cpu().numpy().view(np.uint32), want)


def _pair(M, N, K, b_mn, a_mn=False, seed=0, ragged_ld=False):
    """A, the weight as stored for the F32X3 call, and its planes"""
    import wav2letter_b200 as w

    def rows_padded(t):  # the same matrix with a row stride past its row length, a multiple of 4 floats (a TMA row)
        pad = torch.zeros(t.shape[0], (t.shape[1] + 3) // 4 * 4 + 4, device="cuda")
        pad[:, : t.shape[1]] = t
        return pad[:, : t.shape[1]]

    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn((K, M) if a_mn else (M, K), device="cuda", generator=g)
    Wt = torch.randn((K, N) if b_mn else (N, K), device="cuda", generator=g)
    if ragged_ld:
        A, Wt = rows_padded(A), rows_padded(Wt)
    return A, Wt, w.capi.split_tf32(Wt, transpose=b_mn)


def _both(A, Wt, P, M, N, K, a_mn, b_mn, **kw):
    import wav2letter_b200 as w

    c_bf16 = kw.pop("out_bf16", False)
    dt = torch.bfloat16 if c_bf16 else torch.float32
    init = kw.pop("init", None)
    outs = []
    for kind, B, bmn in (("f32x3", Wt, b_mn), ("f32x3_split_b", P, False)):
        out = torch.full((M, N), float("nan"), device="cuda", dtype=dt) if init is None else init.clone()
        outs.append(w.capi.gemm(A, B, kind, a_mn, bmn, out=out, M=M, N=N, K=K, **kw))
    torch.cuda.synchronize()
    return outs


# forward Y = X W^T (B = W K-major) and data gradient dX = dY W (B = W MN-major, planes of W^T) of each TDS stage and the head
STEP = [(rows, nout, nin, False) for rows, nout, nin in [(9600, 800, 800), (4800, 1120, 1120), (2400, 1440, 1440), (2400, 10000, 1440)]]
STEP += [(rows, nin, nout, True) for rows, nout, nin in [(9600, 800, 800), (4800, 1120, 1120), (2400, 1440, 1440), (2400, 10000, 1440)]]


@pytest.mark.parametrize("M,N,K,b_mn", STEP)
def test_step_shapes_equal_f32x3(M, N, K, b_mn):
    A, Wt, P = _pair(M, N, K, b_mn, seed=M + N)
    ref, got = _both(A, Wt, P, M, N, K, False, b_mn)
    assert not torch.isnan(ref).any()
    assert torch.equal(ref, got)


@pytest.mark.parametrize("M,N,K,b_mn,a_mn,ragged_ld", [
    (1000, 800, 800, False, False, False),   # N = 800: last tile 32 wide; M not a multiple of 128
    (1000, 1440, 10000, True, False, False),  # K = 10000: a k tail of 16 in the last k block
    (333, 100, 75, False, False, True),      # one ragged tile in every direction, K rows padded past the source
    (77, 75, 300, True, False, True),        # transposed planes with a padded K
    (1000, 800, 1000, False, True, False),   # A MN-major
])
def test_ragged_edges_equal_f32x3(M, N, K, b_mn, a_mn, ragged_ld):
    A, Wt, P = _pair(M, N, K, b_mn, a_mn=a_mn, seed=M * 3 + K, ragged_ld=ragged_ld)
    ref, got = _both(A, Wt, P, M, N, K, a_mn, b_mn)
    assert not torch.isnan(ref).any()
    assert torch.equal(ref, got)


@pytest.mark.parametrize("epi", ["bias_relu", "dropout", "aux_relu", "aux_dropout", "accumulate", "bf16_out", "split_k"])
def test_epilogues_equal_f32x3(epi):
    M, N, K = (128, 256, 4096) if epi == "split_k" else (1000, 800, 1120)  # split-K: 2 tiles, 128 k blocks
    A, Wt, P = _pair(M, N, K, False, seed=11)
    kw = {}
    if epi == "bias_relu":
        kw = dict(bias=torch.randn(N, device="cuda"), act=1)
    elif epi == "dropout":
        kw = dict(bias=torch.randn(N, device="cuda"), act=1, dropout_p=0.2, seed=1234)
    elif epi in ("aux_relu", "aux_dropout"):
        aux = torch.relu(torch.randn(M, N, device="cuda"))
        kw = dict(aux=aux, aux_mode=1 if epi == "aux_relu" else 2, aux_scale=1.25)
    elif epi == "accumulate":
        kw = dict(accumulate=True, init=torch.randn(M, N, device="cuda"))
    elif epi == "bf16_out":
        kw = dict(out_bf16=True, bias=torch.randn(N, device="cuda"))
    ref, got = _both(A, Wt, P, M, N, K, False, False, **kw)
    assert not torch.isnan(ref.float()).any()
    assert torch.equal(ref, got)


@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("M,N,K", [(2400, 1440, 1440), (256, 512, 1440)])  # 228 tiles (dynamic schedule), 8 tiles (one wave)
def test_schedules_equal_f32x3(variant, M, N, K):
    import wav2letter_b200 as w

    A, Wt, P = _pair(M, N, K, False, seed=variant + M)
    try:
        w.capi.gemm_set_variant(variant)
        ref, got = _both(A, Wt, P, M, N, K, False, False, bias=torch.randn(N, device="cuda"))
    finally:
        w.capi.gemm_set_variant(1)
    assert torch.equal(ref, got)


def test_split_b_rejects_mn_major_planes():
    import wav2letter_b200 as w

    A, Wt, P = _pair(256, 256, 256, False)
    with pytest.raises(w.capi.W2LError):
        w.capi.gemm(A, P[0], "f32x3_split_b", False, True, M=256, N=256, K=256)
