"""The conv_glu large-channel convolution at the recipes' own shapes, against the float64 model of
tests/conv_glu_reference.py.

1. w2l_conv1d_arrange_ex only moves values: its fp32 / bf16 / fp16 operands must equal the model's bit for bit (16-bit:
   torch's round-to-nearest-even cast, as __float2bfloat16_rn / __float2half_rn), at every (cin, cout, kw) of both conv_glu
   recipes in the padding of every precision mode, and at the kernel's structural edges: kw = 1, even kw (shared-memory
   pitch kw|1), kw 31 / 32 / 33 (the load's index walk steps whole input channels below 32 taps only), kw = 99 (the widest the
   200 KB shared-memory tile admits), partial 32-channel input tiles, odd GLU halves whose 16-channel output tiles straddle
   the two padded halves, and padded sizes above the minimum.  Destinations start as NaN, so a hole in the zero fill or a
   missed write shows.  Rejected arguments return before anything is written.
2. w2l_conv1d_unarrange_grad adds exactly one fp32 addition per weight element and never reads the padding (NaN there);
   its bias gradient is a fixed-order fp32 sum within the bound of its summation depth, also past 64 x 2048 rows where the
   grid stops growing and each CTA strides over more rows.
3. Whole layers through the trainer (fl::Conv2D::forwardGemm: one GEMM over the batch with slack rows between samples):
   emissions and every parameter gradient element by element within the rounding bound of
   conv_glu_reference.ConvGluNet, with the three samples' features scaled by 1e3, 1e-3 and 1 so that a window reaching
   into the neighbouring sample is a thousand-fold error; and a sample's emissions in the batch are the bits it gets alone.
"""
import ctypes

import pytest
import torch

from conv_glu_reference import ConvGluNet, arrange, conv_glu_layers, out_rows, padded_sizes, unarrange

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, scope="module")
def _keep_seed_stream():
    """the trainers built here draw parameter-initialisation seeds from the library's process-wide stream: put it back
    afterwards, so that the tests that follow start from the parameters they would have without this file"""
    from wav2letter_b200 import capi

    seed = capi.lib.w2l_get_seed()
    yield
    capi.lib.w2l_set_seed(seed)

OUT_TYPES = {"f32": (0, torch.float32), "bf16": (1, torch.bfloat16), "fp16": (2, torch.float16)}  # operand type per mode
NAN_BITS = {torch.float32: 0x7FC00001, torch.bfloat16: 0x7FC1, torch.float16: 0x7E01}
INT_VIEW = {torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float16: torch.int16}


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def nan_filled(shape, dtype):
    t = torch.empty(shape, dtype=dtype, device="cuda")
    t.view(INT_VIEW[dtype]).fill_(NAN_BITS[dtype])
    return t


def same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(INT_VIEW[a.dtype]), b.view(INT_VIEW[b.dtype]))


# every (cin, cout, kw) of conv_glu_wsj() and conv_glu_librispeech(), both with NFEAT 40 and 80; all feed a GLU
RECIPE_SHAPES = sorted({(cin, cout, kw) for nfeat in (40, 80) for cin, cout, kw, _ in conv_glu_layers(nfeat)})
# (cin, cout, kw, glu, extra input / output padding beyond the minimum)
EDGE_SHAPES = [(33, 34, 1, True, 0, 0), (33, 34, 2, True, 0, 0), (40, 70, 31, True, 0, 0), (40, 70, 32, True, 0, 0),
               (40, 70, 33, True, 0, 0), (35, 18, 99, True, 0, 0), (1, 30, 5, True, 0, 0), (31, 30, 5, True, 0, 0),
               (32, 30, 5, True, 0, 0), (33, 30, 5, True, 0, 0), (17, 2, 3, True, 0, 0), (37, 26, 7, False, 0, 0),
               (45, 22, 5, True, 8, 16), (45, 21, 3, False, 4, 12)]
ALL_SHAPES = [(cin, cout, kw, True, 0, 0) for cin, cout, kw in RECIPE_SHAPES] + EDGE_SHAPES


def shape_id(s):
    return "cin{}-cout{}-kw{}{}{}".format(s[0], s[1], s[2], "-glu" if s[3] else "", f"-extra{s[4]}x{s[5]}" if s[4] or s[5] else "")


def sizes(kind, cin, cout, glu, xin, xout):
    cin_p, cout_p = padded_sizes(kind, cin, cout, glu)
    return cin_p + xin, cout_p + xout


def run_arrange(w, bias, cin_p, cout_p, glu, mode, flip=True):
    from wav2letter_b200 import capi

    cout, cin, kw = w.shape
    out, dt = OUT_TYPES[mode]
    fwd = nan_filled((cout_p, kw * cin_p), dt)
    fl = nan_filled((cin_p, kw * cout_p), dt) if flip else None
    bias_p = nan_filled((cout_p,), torch.float32) if bias is not None else None
    rc = capi.lib.w2l_conv1d_arrange_ex(torch.cuda.current_stream().cuda_stream, cin, cout, kw, cin_p, cout_p, int(glu), _p(w), _p(bias),
                                        _p(fwd), _p(fl), _p(bias_p), out)
    torch.cuda.synchronize()
    return rc, fwd, fl, bias_p


# ------------------------------------------------------------------------------------------------------------------------
# 1. w2l_conv1d_arrange_ex
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", ALL_SHAPES, ids=shape_id)
def test_arrange_bits(shape):
    cin, cout, kw, glu, xin, xout = shape
    g = torch.Generator(device="cuda").manual_seed(cin * 7919 + cout * 31 + kw)
    w = torch.randn(cout, cin, kw, device="cuda", generator=g)
    bias = torch.randn(cout, device="cuda", generator=g)
    for mode, (_, dt) in OUT_TYPES.items():
        cin_p, cout_p = sizes(mode, cin, cout, glu, xin, xout)
        rc, fwd, flip, bias_p = run_arrange(w, bias, cin_p, cout_p, glu, mode)
        assert rc == 0
        rf, rfl, rb = arrange(w, bias, cin_p, cout_p, glu)  # fp32 moves: exact
        assert same_bits(fwd, rf.to(dt)), f"{mode}: forward operand differs at {int((fwd.float() != rf.to(dt).float()).sum())} entries"
        assert same_bits(flip, rfl.to(dt)), f"{mode}: flipped operand differs at {int((flip.float() != rfl.to(dt).float()).sum())} entries"
        assert same_bits(bias_p, rb), f"{mode}: padded bias differs"


@pytest.mark.parametrize("mode", list(OUT_TYPES))
def test_arrange_without_flip_or_bias(mode):
    """flip = NULL writes the forward operand alone; bias = NULL leaves bias_p to the zero fill"""
    from wav2letter_b200 import capi

    cin, cout, kw, glu = 65, 42, 9, True
    g = torch.Generator(device="cuda").manual_seed(5)
    w = torch.randn(cout, cin, kw, device="cuda", generator=g)
    cin_p, cout_p = sizes(mode, cin, cout, glu, 0, 0)
    _, dt = OUT_TYPES[mode]
    rf, rfl, _ = arrange(w, None, cin_p, cout_p, glu)
    rc, fwd, flip, _ = run_arrange(w, None, cin_p, cout_p, glu, mode, flip=False)
    assert rc == 0 and flip is None and same_bits(fwd, rf.to(dt))
    bias_p = nan_filled((cout_p,), torch.float32)
    fwd = nan_filled((cout_p, kw * cin_p), dt)
    flip = nan_filled((cin_p, kw * cout_p), dt)
    rc = capi.lib.w2l_conv1d_arrange_ex(torch.cuda.current_stream().cuda_stream, cin, cout, kw, cin_p, cout_p, 1, _p(w), None, _p(fwd),
                                        _p(flip), _p(bias_p), OUT_TYPES[mode][0])
    torch.cuda.synchronize()
    assert rc == 0 and same_bits(fwd, rf.to(dt)) and same_bits(flip, rfl.to(dt))
    assert same_bits(bias_p, torch.zeros_like(bias_p))


@pytest.mark.parametrize("case", ["kw100", "odd_glu_cout", "glu_cout_p_not_x8", "out_type_3"])
def test_arrange_rejections_write_nothing(case):
    from wav2letter_b200 import capi

    cin, cout, kw, glu, cout_p, out, code = {"kw100": (8, 8, 100, 1, 8, 0, capi.W2L_ERR_UNSUPPORTED),
                                             "odd_glu_cout": (8, 7, 3, 1, 8, 0, capi.W2L_ERR_INVALID_ARGUMENT),
                                             "glu_cout_p_not_x8": (8, 6, 3, 1, 12, 0, capi.W2L_ERR_INVALID_ARGUMENT),
                                             "out_type_3": (8, 8, 3, 1, 8, 3, capi.W2L_ERR_INVALID_ARGUMENT)}[case]
    w = torch.randn(cout, cin, kw, device="cuda")
    bias = torch.randn(cout, device="cuda")
    fwd = nan_filled((cout_p, kw * cin), torch.float32)
    flip = nan_filled((cin, kw * cout_p), torch.float32)
    bias_p = nan_filled((cout_p,), torch.float32)
    torch.cuda.synchronize()
    launches = capi.launch_count()
    rc = capi.lib.w2l_conv1d_arrange_ex(torch.cuda.current_stream().cuda_stream, cin, cout, kw, cin, cout_p, glu, _p(w), _p(bias), _p(fwd),
                                        _p(flip), _p(bias_p), out)
    torch.cuda.synchronize()
    assert rc == code, capi.lib.w2l_last_error().decode()
    assert capi.launch_count() == launches
    for t in (fwd, flip, bias_p):
        assert same_bits(t, nan_filled(t.shape, torch.float32)), "a rejected call wrote its destination"
    if case == "kw100":
        dw = torch.zeros_like(w)
        rc = capi.lib.w2l_conv1d_unarrange_grad(torch.cuda.current_stream().cuda_stream, cin, cout, kw, cin, cout_p, glu, _p(fwd), _p(dw), 0,
                                                None, None)
        torch.cuda.synchronize()
        assert rc == capi.W2L_ERR_UNSUPPORTED and capi.launch_count() == launches and not dw.count_nonzero()


# ------------------------------------------------------------------------------------------------------------------------
# 2. w2l_conv1d_unarrange_grad
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", ALL_SHAPES, ids=shape_id)
def test_unarrange_bits(shape):
    """dw += unarrange(dfwd): one fp32 addition per element, in the padding of the f32 / tf32 and the bf16 / fp16 modes"""
    from wav2letter_b200 import capi

    cin, cout, kw, glu, xin, xout = shape
    g = torch.Generator(device="cuda").manual_seed(cin * 104729 + cout * 13 + kw)
    for kind in ("f32", "bf16"):
        cin_p, cout_p = sizes(kind, cin, cout, glu, xin, xout)
        dfwd = torch.full((cout_p, kw, cin_p), float("nan"), device="cuda")
        rows = out_rows(cout, cout_p, glu, "cuda")
        dfwd[rows, :, :cin] = torch.randn(cout, kw, cin, device="cuda", generator=g)
        dfwd = dfwd.view(cout_p, kw * cin_p)
        dw = torch.randn(cout, cin, kw, device="cuda", generator=g)
        want = dw + unarrange(dfwd, cin, cout, kw, cin_p, cout_p, glu)
        rc = capi.lib.w2l_conv1d_unarrange_grad(torch.cuda.current_stream().cuda_stream, cin, cout, kw, cin_p, cout_p, int(glu), _p(dfwd),
                                                _p(dw), 0, None, None)
        torch.cuda.synchronize()
        assert rc == 0
        assert same_bits(dw, want), f"{kind}: {int((dw != want).sum())} of {dw.numel()} weight-gradient elements differ"


def bias_grad_depth(rows):
    """additions on the longest path of w2l_conv1d_unarrange_grad's bias sum: a thread's rows (grid.y CTAs of 8 row
    threads, grid.y = min(ceil(rows / 2048), 64)), the 8 row threads of a CTA, the grid.y partials, the add onto dbias"""
    gy = min((rows + 2047) // 2048, 64)
    return (rows + 8 * gy - 1) // (8 * gy) + 8 + gy + 1


@pytest.mark.parametrize("rows", [1, 8, 2047, 2048, 2049, 131072, 131073, 500000])
@pytest.mark.parametrize("cout,glu", [(70, True), (37, False)])
def test_bias_grad(rows, cout, glu):
    """|dbias - ref| <= gamma_n (|dbias0| + sum |dy|) per channel, n the summation depth (Higham's gamma_n = n u / (1 - n u));
    NaN in dy's padded columns never reaches dbias; two runs give the same bits"""
    from wav2letter_b200 import capi

    cin, kw = 4, 1
    cin_p, cout_p = sizes("bf16", cin, cout, glu, 0, 0)
    g = torch.Generator(device="cuda").manual_seed(rows + cout)
    chans = out_rows(cout, cout_p, glu, "cuda")
    dy = torch.full((rows, cout_p), float("nan"), device="cuda")
    dy[:, chans] = torch.randn(rows, cout, device="cuda", generator=g) + 0.5  # an offset, so the sums do not cancel to nothing
    dfwd = torch.randn(cout_p, kw * cin_p, device="cuda", generator=g)
    dbias0 = torch.randn(cout, device="cuda", generator=g)

    def run(dy_, with_dbias=True):
        dw, db = torch.zeros(cout, cin, kw, device="cuda"), dbias0.clone()
        rc = capi.lib.w2l_conv1d_unarrange_grad(torch.cuda.current_stream().cuda_stream, cin, cout, kw, cin_p, cout_p, int(glu), _p(dfwd),
                                                _p(dw), rows, _p(dy_), _p(db) if with_dbias else None)
        torch.cuda.synchronize()
        assert rc == 0
        assert same_bits(dw, unarrange(dfwd, cin, cout, kw, cin_p, cout_p, glu)), "the weight part of the call went wrong"
        return db

    db = run(dy)
    sel = dy[:, chans].double()
    ref = dbias0.double() + sel.sum(0)
    n = bias_grad_depth(rows)
    gamma = n * 2.0 ** -24 / (1 - n * 2.0 ** -24)  # measured on an H100 80GB HBM3 (700 W): at most 0.19 of this bound
    bound = gamma * (dbias0.double().abs() + sel.abs().sum(0))
    ratio = float(((db.double() - ref).abs() / bound).max())
    print(f"rows {rows} cout {cout}: max |err| / bound {ratio:.3g}")
    assert ratio <= 1.0, ratio
    assert same_bits(run(dy), db), "the bias gradient changed between two runs"
    assert same_bits(run(None), dbias0), "dy = NULL must leave dbias untouched"
    # dbias = NULL: the weight gradient alone (checked in run); neither dy nor a bias buffer anywhere else changes
    dy0 = dy.clone()
    assert same_bits(run(dy, with_dbias=False), dbias0) and same_bits(dy, dy0)


# ------------------------------------------------------------------------------------------------------------------------
# 3. whole layers through the trainer
# ------------------------------------------------------------------------------------------------------------------------
N_LABEL = 6
SCALES = (1e3, 1e-3, 1.0)
# name -> (layers (cin, cout, kw, pad), feature count, T values): conv outputs of 1 frame, a few, and several hundred.
# The input view needs a feature count that is a multiple of 8; the 683-channel layer reads the first 683 of 688 features
# (its operand is padded to 688 input channels in every precision mode, past f32's minimum of 684).  The 170-frame padding
# of the LibriSpeech first layer turns a 1-frame utterance into 329 output frames (316 after the second layer), more than
# Trainer.forward's first guess of 2 T + 64 frames per sample.
LAYER_CASES = {
    "librispeech_683_1502_27": ([(683, 1502, 27, 0)], 688, (27, 30, 300)),
    "librispeech_first_pad170": ([(80, 400, 13, 170)], 80, (1, 300)),
    "librispeech_first_two": ([(80, 400, 13, 170), (200, 440, 14, 0)], 80, (1, 260)),
    "wsj_200_450_10_pad0": ([(200, 450, 10, 0)], 200, (10, 13, 400)),
}
# the bounds of ConvGluNet are first order: products of two error terms (relative size c^2) are left out, and the factor
# 1.25 covers them
FIRST_ORDER_SLACK = 1.25


def arch_text(layers):
    out = ["V -1 1 NFEAT 0"]
    for cin, cout, kw, pad in layers:
        out += [f"WN 3 C {cin} {cout} {kw} 1 {pad}", "GLU 2", "DO 0.0"]
    out += ["RO 2 0 3 1", f"WN 0 L {layers[-1][1] // 2} NLABEL"]
    return "\n".join(out) + "\n"


def layer_params():
    for name, (layers, nfeat, Ts) in LAYER_CASES.items():
        for T in Ts:
            for precision in ("f32", "tf32", "bf16", "fp16"):
                yield pytest.param(name, T, precision, id=f"{name}-T{T}-{precision}")


def ratio_of(got, want, bound):
    return float(((got.double() - want).abs() / (FIRST_ORDER_SLACK * bound + 1e-300)).max())


@pytest.mark.parametrize("name,T,precision", list(layer_params()))
def test_layers_through_trainer(name, T, precision):
    import wav2letter_b200 as w2l
    from wav2letter_b200.trainer import Trainer

    layers, nfeat, _ = LAYER_CASES[name]
    B = len(SCALES)
    tr = Trainer(arch_text(layers), nfeat, N_LABEL, "asg", "target_sz_sqrt", transdiag=1.0, lr=0.0, lrcrit=0.0, precision=precision)
    g = torch.Generator(device="cuda").manual_seed(11 + T)
    feat = torch.randn((B, 1, nfeat, T), device="cuda", generator=g) * torch.tensor(SCALES, device="cuda").view(B, 1, 1, 1)
    flat0 = tr.get_flat(0, 0).clone()
    emis = tr.forward(feat).clone()
    Tout = emis.shape[1]
    L = min(3, Tout)
    tgt = torch.randint(0, N_LABEL, (B, L), device="cuda", generator=g, dtype=torch.int32)
    # the criterion's own gradient of these emissions: the trainer's step (total batch 1: no rescaling) starts from it
    trans = tr.get_flat(1, 0).view(N_LABEL, N_LABEL)
    _, G, _ = w2l.asg_forward_backward(emis, tgt, trans, "target_sz_sqrt")
    tr.step(feat, tgt, train=True, total_batch=1.0)
    torch.cuda.synchronize()
    grads = tr.get_flat(0, 1)
    layout = tr.layout(0)
    params = [flat0[off:off + n].double() for off, n, _ in layout]
    net = ConvGluNet(params, layers, precision)
    z, Ez = net.forward(feat.double()[:, 0, :layers[0][0]])
    assert z.shape == emis.shape, (z.shape, emis.shape)
    worst = {}
    for b in range(B):
        r = ratio_of(emis[b], z[b], Ez[b])
        worst[f"emissions[{b}]"] = r
    ref = net.backward(G.double())
    names = [f"layer{i}.{p}" for i in range(len(layers)) for p in ("v", "g", "bias")] + ["head.v", "head.g", "head.bias"]
    for nm, (off, n, _), (d, E) in zip(names, layout, ref):
        worst[nm] = ratio_of(grads[off:off + n], d, E)
    print(f"{name} T={T} T'={Tout} {precision}: max |err| / bound " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    bad = {k: v for k, v in worst.items() if not v <= 1.0}
    assert not bad, f"beyond the rounding bound: {bad}"

    # each sample alone at the same T: the same windows, the same GEMM sums in the same order (no split-K with a bias)
    for b in range(B):
        alone = tr.forward(feat[b:b + 1].contiguous())
        assert same_bits(alone[0], emis[b]), f"sample {b}: batched emissions differ from the sample alone at " \
                                             f"{int((alone[0] != emis[b]).sum())} of {emis[b].numel()} entries"
