"""The persistent GEMM's dynamic tile schedule and the trainer's gradient stream.

The persistent kernel hands out work items (tile, split-K slice) from a per-stream counter, so which CTA computes which
tile depends on timing; every item still keeps its k order and its split-K slice, so results must equal the
one-tile-per-CTA kernel's bit for bit, alone, next to a GEMM on another stream, and launch after launch (the counter is
reset by the last CTA of each launch).  The trainer computes the Linear weight gradients on a second stream; losses and
parameters must not change by a bit whether it does or not, also when the gradient stream is held back by a delay
kernel before each piece of work (a missing wait or an early free then shows up as a mismatch)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# 2400 x 1440 x 1440: 19 x 12 = 228 tiles, more than one wave, so the counter hands out tiles; 128 x 128 x 800: one tile
# split six ways in slices of 5 k blocks, the last one empty (6 items, one wave: the walk ends on the first claim)
SHAPES = [(2400, 1440, 1440), (304, 10000, 1440), (128, 128, 800)]


def _operands(M, N, K, a_mn, b_mn, kind, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn((K, M) if a_mn else (M, K), device="cuda", generator=g)
    B = torch.randn((K, N) if b_mn else (N, K), device="cuda", generator=g)
    if kind == "bf16":
        A, B = A.bfloat16(), B.bfloat16()
    return A, B


def _gemm(w, A, B, kind, a_mn, b_mn, bias=None):
    M, K = (A.shape[1], A.shape[0]) if a_mn else A.shape
    N = B.shape[1] if b_mn else B.shape[0]
    out = torch.full((M, N), float("nan"), device="cuda")  # a tile nobody computed stays NaN
    return w.capi.gemm(A, B, kind, a_mn, b_mn, bias=bias, act=0 if bias is None else 1, out=out)


@pytest.mark.parametrize("kind", ["f32x3", "tf32", "bf16"])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_dynamic_schedule_matches_per_tile_kernel(M, N, K, a_mn, b_mn, kind):
    import wav2letter_b200 as w

    A, B = _operands(M, N, K, a_mn, b_mn, kind, seed=M + N + K)
    bias = torch.randn(N, device="cuda")
    try:
        w.capi.gemm_set_variant(0)
        C0, P0 = _gemm(w, A, B, kind, a_mn, b_mn, bias), _gemm(w, A, B, kind, a_mn, b_mn)
        w.capi.gemm_set_variant(1)
        C1, P1 = _gemm(w, A, B, kind, a_mn, b_mn, bias), _gemm(w, A, B, kind, a_mn, b_mn)
    finally:
        w.capi.gemm_set_variant(1)
    torch.cuda.synchronize()
    assert not torch.isnan(P0).any()
    assert torch.equal(C0, C1)
    assert torch.equal(P0, P1)


@pytest.mark.parametrize("kind", ["f32x3", "bf16"])
def test_two_streams_concurrently(kind):
    """a TDS stage-3 backward pair: the weight gradient (both operands MN-major) on one stream, the data gradient on the
    other, launched together several times; each result equals its serial one"""
    import wav2letter_b200 as w

    Aw, Bw = _operands(1440, 1440, 2400, True, True, kind, seed=1)
    Ad, Bd = _operands(2400, 1440, 1440, False, True, kind, seed=2)
    ref_w = _gemm(w, Aw, Bw, kind, True, True)
    ref_d = _gemm(w, Ad, Bd, kind, False, True)
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs = []
    for _ in range(4):
        with torch.cuda.stream(s1):
            cw = _gemm(w, Aw, Bw, kind, True, True)
        with torch.cuda.stream(s2):
            cd = _gemm(w, Ad, Bd, kind, False, True)
        outs.append((cw, cd))
    torch.cuda.synchronize()
    for cw, cd in outs:
        assert torch.equal(cw, ref_w)
        assert torch.equal(cd, ref_d)


def test_back_to_back_launches_on_one_stream():
    """each launch starts from a reset counter: a stale count would skip tiles (left NaN) or repeat them"""
    import wav2letter_b200 as w

    shapes = [(2400, 1440, 1440, False, True), (4800, 1120, 1120, False, False), (304, 10000, 1440, False, False)]
    ops = [_operands(M, N, K, a, b, "f32x3", seed=M) for M, N, K, a, b in shapes]
    try:
        w.capi.gemm_set_variant(0)
        refs = [_gemm(w, A, B, "f32x3", a, b) for (A, B), (_, _, _, a, b) in zip(ops, shapes)]
    finally:
        w.capi.gemm_set_variant(1)
    got = [_gemm(w, A, B, "f32x3", a, b) for _ in range(3) for (A, B), (_, _, _, a, b) in zip(ops, shapes)]
    torch.cuda.synchronize()
    for i, C in enumerate(got):
        assert torch.equal(C, refs[i % len(shapes)]), f"launch {i}"


ARCH = """V -1 NFEAT 1 0
C2 1 4 5 1 2 1 -1 -1
R
LN 3
TDS 4 5 80 0.0
C2 4 8 5 1 2 1 -1 -1
R
LN 3
TDS 8 5 80 0.0
TDS 8 5 80 0.0
V 0 640 1 0
RO 1 0 3 2
L 640 NLABEL
"""


@pytest.mark.parametrize("delay_us", [0, 2000])
@pytest.mark.parametrize("precision", ["f32", "bf16"])
def test_trainer_grad_stream_on_and_off_agree(precision, delay_us):
    from wav2letter_b200.trainer import Trainer

    N, B, T, L = 30, 16, 1200, 40
    trainers = [Trainer(ARCH, 80, N, "ctc", "target_sz", lr=0.05, momentum=0.5, maxgradnorm=1.0, precision=precision) for _ in range(2)]
    on, off = trainers
    off.set_grad_stream(False)
    on.set_grad_stream_delay(delay_us)
    off.set_flat(on.get_flat(0, 0), 0)
    g = torch.Generator(device="cuda").manual_seed(5)
    losses = {0: [], 1: []}
    for step in range(3):
        feat = torch.randn((B, 1, 80, T), device="cuda", generator=g)
        tgt = torch.randint(0, N - 1, (B, L), device="cuda", generator=g, dtype=torch.int32)
        tgt[::3, L // 2:] = -1
        for k, tr in enumerate(trainers):
            losses[k].append(tr.step(feat, tgt, train=True).clone())
    torch.cuda.synchronize()
    for a, b in zip(losses[0], losses[1]):
        assert torch.isfinite(a).all()
        assert torch.equal(a, b)
    assert torch.equal(on.get_flat(0, 0), off.get_flat(0, 0))
    assert torch.equal(on.get_flat(0, 1), off.get_flat(0, 1))
    for tr in trainers:
        tr.close()
