"""LayerNorm where a one-pass variance cancels: every LayerNorm kernel against float64 torch at large mean / sigma, at a
variance near and below eps, on constant groups, on a group whose first value is an outlier, on post-ReLU rows and at
tiny group sizes.

The reference is float64 torch on the values the kernels normalise: x = a + r added in fp32, then promoted, so the
residual add is not counted against the kernels.  No fp32 kernel beats fp32 rounding (the stored mean alone is rounded
to fp32), so each error is measured against what stock fp32 torch (F.layer_norm and its autograd on the same fp32 x)
makes of the same inputs: a kernel passes within 4x of that or within 2e-6, whichever is larger.  The scalar gain and
bias gradients are held to 1e-4 relative, or 4x torch's where its own error is larger; at mean / sigma >= 1e3 the fp32
mean the forward stores moves every xhat by up to half an ulp of the mean, and twice what that rounding alone does to the
gain gradient is allowed too.  Well-conditioned cases (mean / sigma <= 1, post-ReLU rows) also keep the absolute bounds
of test_gpu_am_kernels.py, and constant groups must come out exactly `bias`.

Every case asserts, via capi.trace, the kernels it ran: the one-warp-per-group forward and backward (V = 4 and V = 1), the
w2l_layernorm_rows_fwd entry point with few groups, the two-pass forward and backward (V = 4 and V = 1), and the
cooperative single-launch forward at chunks larger than its shared-memory copy, so that its tail is read back from L2.
V = 1 is forced by row lengths that are not multiples of 4 and by buffers that start one float into their allocation."""
import zlib

import pytest
import torch
import torch.nn.functional as F

from test_gpu_trainer import PREC_TOL, STREAMING_ARCH, TorchStreamingTDS, make_batch

pytestmark = pytest.mark.gpu

EPS = 1e-5
FUSED_KEEP = 110 * 1024 // 4  # floats of a chunk that ln_fused_fwd_kernel keeps in shared memory (kLnFusedSmem / 4)
TWO_PASS_BWD = {"ln_bwd_stats_kernel", "ln_bwd_apply_kernel", "ln_scalar_grads_kernel"}
ROWS_BWD = {"ln_row_bwd_kernel", "ln_scalar_grads_kernel"}
# name -> (groups, R, buffer offset in floats, forward kernels, backward kernels (None: a forward-only entry point))
FAMILIES = {
    "rows_v4": (2400, 640, 0, {"ln_row_fwd_kernel"}, ROWS_BWD),  # ln_use_rows: groups * 32 >= SMs * 256
    "rows_v1": (2400, 642, 1, {"ln_row_fwd_kernel"}, ROWS_BWD),
    "rows_entry_v4": (6, 640, 0, {"ln_row_fwd_kernel"}, None),  # w2l_layernorm_rows_fwd: the streaming model's few frames
    "rows_entry_v1": (6, 642, 1, {"ln_row_fwd_kernel"}, None),
    "two_pass_v4": (3, 5000, 0, {"ln_stats_kernel", "ln_apply_kernel"}, TWO_PASS_BWD),
    "two_pass_v1": (3, 5002, 1, {"ln_stats_kernel", "ln_apply_kernel"}, TWO_PASS_BWD),
    "fused": (128, 80000, 0, {"ln_fused_fwd_kernel"}, TWO_PASS_BWD),
}
# (kind, value): mean / sigma of x; sigma^2 around eps (mean 1); every value of a group equal to `value`; a group whose
# first value sits 50 sigma above the mean (the pivot must not follow it); post-ReLU values, half of them zeros (skewed,
# well-conditioned: kept on the plain sums, which are accurate there)
CONDITIONS = ([("ratio", v) for v in (0.0, 30.0, 100.0, 1e3, 1e4)] + [("var", v) for v in (1e-3, 1e-5, 1e-7)]
              + [("const", v) for v in (17.7, 3.3, -250.1, 0.0)] + [("outlier", v) for v in (0.0, 100.0)] + [("relu", 1.3)])


def rel(a, b):
    a, b = a.detach(), b.detach()
    return float((a.double() - b.double()).abs().max() / max(1e-6, float(b.double().abs().max())))


def shifted(t, off):
    """a copy of t that starts `off` floats into its allocation"""
    buf = torch.empty(t.numel() + off, device=t.device, dtype=t.dtype)
    out = buf[off:].view(t.shape)
    out.copy_(t)
    return out


def make_inputs(cond, G, R, res, seed):
    """(a, r): a branch output a and a residual r (None without one) whose fp32 sum has the condition `cond`"""
    kind, v = cond
    gen = torch.Generator(device="cuda").manual_seed(seed)
    noise = lambda: torch.randn((G, R), device="cuda", generator=gen, dtype=torch.float64)  # noqa: E731
    if kind == "const":  # with a residual, x = fl(0.5 + v): constant too
        a = torch.full((G, R), 0.5 if res else v, device="cuda", dtype=torch.float64)
        return a.float(), torch.full((G, R), v, device="cuda").float() if res else None
    if kind == "relu":
        return (noise().clamp_min(0) * v).float(), (noise().clamp_min(0) * 0.7).float() if res else None
    mean, sd = (1.0, v ** 0.5) if kind == "var" else (v, 1.0)
    z = noise() * sd
    if kind == "outlier":
        z[:, 0] = 50 * sd
    if not res:
        return (mean + z).float(), None
    return (noise().clamp_min(0) * 0.5 * sd).float(), (mean + z).float()  # a post-ReLU branch: it has zeros for the mask


def rows_fwd(a, r, gain, bias):
    """w2l_layernorm_rows_fwd, the one-warp-per-group forward whatever the group count"""
    from wav2letter_b200 import capi

    G, R = a.shape
    y, mr = torch.empty_like(a), torch.empty((G, 2), device="cuda")
    capi._check(capi.lib.w2l_layernorm_rows_fwd(capi._stream(), G, R, EPS, capi._ptr(a), capi._ptr(r), capi._ptr(gain), capi._ptr(bias),
                                                capi._ptr(y), capi._ptr(mr)))
    return y, mr


def run_kernels(family, a, r, dy, gain, bias, branch_mode):
    """forward and backward of `family` on (a, r), asserting the kernels that ran"""
    from wav2letter_b200 import capi

    _, _, _, fwd_kernels, bwd_kernels = FAMILIES[family]
    out = {}
    fwd = rows_fwd if family.startswith("rows_entry") else capi.layernorm_fwd
    ran = capi.trace(lambda: out.update(zip(("y", "mr"), fwd(a, r, gain, bias))))
    assert set(ran) == fwd_kernels, (family, ran)
    if bwd_kernels is not None:
        ran = capi.trace(lambda: out.update(zip(("d_branch", "d_res", "dgain", "dbias"),
                                                capi.layernorm_bwd(a, r, dy, gain, out["mr"], branch_mode, 1.25))))
        assert set(ran) == bwd_kernels, (family, ran)
    return out


def layer_norm_graph(x, gain, bias, dy, dtype):
    """y = F.layer_norm(x) * gain + bias in `dtype` and the gradients of dy . y: (y, dx, dgain, dbias)"""
    x, g, b = (t.detach().to(dtype).requires_grad_(True) for t in (x, gain, bias))
    y = F.layer_norm(x, x.shape[1:], eps=EPS) * g + b
    y.backward(dy.to(dtype))
    return y.detach(), x.grad, g.grad, b.grad


def check_case(family, cond, res, branch_mode=0, R=None, seed_tag=""):
    G, R_family, off, _, bwd_kernels = FAMILIES[family]
    R = R_family if R is None else R
    seed = zlib.crc32(f"{family}/{cond}/{res}/{R}/{seed_tag}".encode())
    a, r = make_inputs(cond, G, R, res, seed)
    dy = torch.randn((G, R), device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed + 1))
    gain, bias = torch.tensor([1.7], device="cuda"), torch.tensor([-0.3], device="cuda")
    if off:
        a, r, dy = shifted(a, off), None if r is None else shifted(r, off), shifted(dy, off)
    x = a + r if r is not None else a  # the fp32 values the kernels normalise
    got = run_kernels(family, a, r, dy, gain, bias, branch_mode)
    y64, dx64, dg64, db64 = layer_norm_graph(x, gain, bias, dy, torch.float64)
    y32, dx32, dg32, db32 = layer_norm_graph(x, gain, bias, dy, torch.float32)
    tag = (family, cond, res, R)
    const = cond[0] == "const"
    well = cond[0] == "relu" or (cond[0] == "ratio" and cond[1] <= 1.0)

    # statistics: the mean within one fp32 ulp plus 2e-6 sigma, rstd within 2e-6 relative of 1 / sqrt(var + eps)
    x64 = x.double()
    mean64, var64 = x64.mean(1), x64.var(1, correction=0)
    mu, rstd = got["mr"][:, 0].double(), got["mr"][:, 1].double()
    mean_err = float(((mu - mean64).abs() / (2.0 ** -23 * mean64.abs() + 2e-6 * var64.sqrt() + 1e-30)).max())
    rstd_err = float(((rstd - 1 / (var64 + EPS).sqrt()) * (var64 + EPS).sqrt()).abs().max())
    assert mean_err <= 1.0 and rstd_err <= 2e-6, (tag, mean_err, rstd_err)

    # forward
    err, ref_err = rel(got["y"], y64), rel(y32, y64)
    assert err <= max(4 * ref_err, 2e-6), (tag, "y", err, ref_err)
    if well:
        assert err < 1e-5, (tag, err)
    if const or R == 1:
        assert torch.equal(got["y"], bias.expand_as(got["y"])), (tag, got["y"])
    if const:
        assert torch.equal(got["mr"][:, 0], x[:, 0]), tag
        assert float((got["mr"][:, 1].double() * EPS ** 0.5 - 1).abs().max()) <= 1e-6, (tag, got["mr"][:, 1])
    if bwd_kernels is None:
        return got

    # backward: torch's fp32 graph of a constant group normalises its own rounding residue, so there float64 alone sets the bar
    mask = (a > 0).double() * 1.25 if branch_mode == 1 else 1.0
    for name, ref, ref32 in (("d_res", dx64, dx32), ("d_branch", dx64 * mask, dx32.double() * mask)):
        err, ref_err = rel(got[name], ref), rel(ref32, ref)
        assert err <= (2e-6 if const else max(4 * ref_err, 2e-6)), (tag, name, err, ref_err)
        if well:
            assert err < 2e-5, (tag, name, err)
    # the gain gradient sums dy * xhat, and xhat is formed from the fp32 mean and rstd the forward stored: where rounding
    # the float64 statistics to fp32 alone moves that sum by more than 1e-4 (mean / sigma >= 1e3), twice that sets the bar
    xhat_f32_stats = (x64 - mean64.float().double()[:, None]) * (1 / (var64 + EPS).sqrt()).float().double()[:, None]
    floor = rel((dy.double() * xhat_f32_stats).sum().view(1), dg64)
    for name, ref, ref32, limit in (("dgain", dg64, dg32, max(1e-4, 2 * floor)), ("dbias", db64, db32, 1e-4)):
        err, ref_err = rel(got[name], ref), rel(ref32, ref)
        assert err <= (limit if const else max(4 * ref_err, limit)), (tag, name, err, ref_err, floor)
    return got


def cond_id(c):
    return f"{c[0]}={c[1]:g}"


@pytest.mark.parametrize("res", [True, False], ids=["residual", "no_residual"])
@pytest.mark.parametrize("cond", CONDITIONS, ids=cond_id)
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_layernorm_conditioning(family, cond, res):
    if family == "fused":
        # ln_fused_fwd_kernel holds at most two CTAs per SM (about 110 KB of shared memory each), so a sample is cut into at
        # most 2 * SMs / groups chunks: each of them longer than what the kernel keeps in shared memory
        G, R = FAMILIES[family][:2]
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        assert R / max(1, 2 * sms // G) > FUSED_KEEP, sms
    check_case(family, cond, res)


@pytest.mark.parametrize("res", [True, False], ids=["residual", "no_residual"])
@pytest.mark.parametrize("R", [1, 2, 3, 5])
@pytest.mark.parametrize("family", ["rows_v1", "two_pass_v1", "rows_entry_v1"])
def test_layernorm_tiny_groups(family, R, res):
    """groups of 1, 2, 3 and 5 values (one value: xhat = 0, the output is `bias` and rstd = 1 / sqrt(eps))"""
    check_case(family, ("ratio", 30.0), res, R=R)


@pytest.mark.parametrize("cond", [("ratio", 0.0), ("ratio", 1e3)], ids=cond_id)
@pytest.mark.parametrize("family", ["rows_v4", "rows_v1", "two_pass_v4", "two_pass_v1"])
def test_layernorm_branch_mask(family, cond):
    """branch mode 1: d_branch = d_res * (a > 0) * scale, on a well- and a badly-conditioned group"""
    check_case(family, cond, True, branch_mode=1)


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_layernorm_run_to_run_bits(family):
    first = check_case(family, ("ratio", 1e3), True, seed_tag="bits")
    again = check_case(family, ("ratio", 1e3), True, seed_tag="bits")
    for k in first:
        assert torch.equal(first[k], again[k]), (family, k)


def tds_ln_input(p, feat):
    """float64 input of the first TDS block's first LayerNorm in TorchStreamingTDS (parameters p in module order)"""
    x = feat.double().permute(0, 3, 1, 2)  # [B,T,1,F]

    def conv(x, w, b, cin, cout, k, s, pl, pr):
        xin = F.pad(x.permute(0, 2, 1, 3), (0, 0, pl, pr))
        return F.conv2d(xin, w.view(cout, cin, k).unsqueeze(-1), b.view(cout), stride=(s, 1)).permute(0, 2, 1, 3)

    x = conv(x, p[0], p[1], 1, 4, 10, 2, 5, 3).clamp_min(0)
    x = F.layer_norm(x, x.shape[2:], eps=EPS) * p[2] + p[3]
    return x + conv(x, p[4], p[5], 4, 4, 9, 1, 7, 1).clamp_min(0)


def test_streaming_train_step_with_a_large_layernorm_mean():
    """One f32 train step of the streaming TDS arch whose first TDS block normalises frames with mean / sigma >= 1000: the
    first LayerNorm's bias is 2000 and that block's time convolution is scaled by 1e-3, so the residual (mean 2000, sigma
    about 1) dominates the block's LayerNorm input.  (A large bias alone would not do: a full-size convolution of an input
    near 2000 gives every channel its own offset, and the frame's sigma grows with it.)  Emissions, loss and every
    parameter gradient against float64 under the f32 criteria of test_gpu_trainer.py; 4 x 400 frames are enough groups
    for the one-warp-per-frame kernels.  Summed without a pivot, their fp32 sums put the emissions 1.3e-3 off (H100)."""
    import oracle
    from wav2letter_b200.trainer import Trainer

    B, T, L, N = 4, 800, 5, 12
    tol = PREC_TOL["f32"]
    tr = Trainer(STREAMING_ARCH, 80, N, "ctc", "target_sz", lr=0.0, lrcrit=0.0, precision="f32")
    layout = tr.layout(0)
    flat = tr.get_flat(0, 0).clone()
    # module order: first convolution (weight, bias), first LayerNorm (gain, bias), the TDS block's convolution (weight, bias)
    ln_bias, (cw, ncw, _), (cb, ncb, _) = layout[3][0], layout[4], layout[5]
    assert layout[3][1] == 1 and ncw == 4 * 4 * 9 and ncb == 4, layout[:6]
    flat[ln_bias] = 2000.0
    flat[cw:cw + ncw] *= 1e-3
    flat[cb:cb + ncb] *= 1e-3
    tr.set_flat(flat)
    feat, tgt = make_batch(B, T, N, L, 7, True)
    loss = tr.step(feat, tgt, train=True)
    grads = tr.get_flat(0, 1)
    got = tr.forward(feat)
    torch.cuda.synchronize()
    ref = TorchStreamingTDS(flat, layout)
    with torch.no_grad():
        s = tds_ln_input(ref.p, feat)
        ratio = s.mean((2, 3)) / s.std((2, 3), correction=0)
    assert float(ratio.min()) >= 1000, float(ratio.min())
    logits = ref.forward(feat)
    ol, ode = oracle.ctc(logits.detach().float().cpu().numpy(), tgt.cpu().numpy(), "target_sz")
    assert rel(got, logits) < tol["emis"], rel(got, logits)
    assert rel(loss, torch.from_numpy(ol).cuda()) < tol["emis"], (loss, ol)
    logits.backward(torch.from_numpy(ode).double().cuda())
    full = torch.cat([p.grad.flatten() for p in ref.p])
    mine = torch.cat([grads[off:off + n] for off, n, _ in layout])
    gscale = float(full.abs().max())
    for (off, n, dims), p in zip(layout, ref.p):
        denom = max(float(p.grad.norm()), tol["floor"] * gscale * n ** 0.5)
        gerr = float((grads[off:off + n].double() - p.grad.flatten()).norm()) / denom
        assert gerr < tol["per_param"], f"param at {off} dims {dims}: grad rel err {gerr}"
    assert rel(mine, full) < tol["overall"], rel(mine, full)
    tr.close()
