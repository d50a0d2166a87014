"""End-to-end parity on the reference's own arch files (BASELINE.json configs[0..3]): forward emissions, criterion loss
and EVERY parameter gradient of one train step of the CUDA path against a float64 torch graph of the same arch
(oracle/am_ref.py) + the C oracle criterion, at reduced T / B.

The arch text comes from wav2letter_b200/archs.py, whose generators tests/test_archs.py checks token-for-token against
recipes/conv_glu/{wsj,librispeech}/network.arch, recipes/seq2seq_tds/librispeech/network.arch and
recipes/streaming_convnets/librispeech/am_500ms_future_context.arch (stored in tests/golden/reference_archs.json).  Dropout probabilities are set to 0 and SpecAugment's mask counts to 0 — random masks cannot be
compared across implementations; both are covered by their own tests.

Tolerances.  precision "f32" (fp32-accurate contractions: 3xTF32 split GEMMs, fp32 SIMT time convolutions):
emissions 2e-4 of the largest emission, per-sample loss 2e-4 (both ~2e-5 / 1e-6 measured), all gradients together within
1e-2 of the largest entry, and every single parameter's gradient within 5e-2 RELATIVE L2 error (floor: 1e-2 of the net's
largest entry) OR within 8x of the error stock fp32 torch (TF32 off) makes on that same parameter against float64.  Two fp32 effects set that floor: the
scalar LayerNorm gains / biases of the TDS archs are sums with heavy cancellation (percent-level noise for ANY fp32
implementation), and at these reduced sizes a Linear sees 40 rows, so a single ReLU whose pre-activation (|pre| < 1e-5)
changes sign between two correct fp32 evaluations moves entries of the next weight gradient by percents (and, through the
cancelling sums, the LayerNorm scalars upstream by more).  Each case appends its measured errors to
w2l_arch_parity.jsonl in the temporary directory.  A wrong gradient formula fails all of this by orders of magnitude.  "tf32" / "bf16" run the same graph with 10- / 8-bit operand mantissas; they
are checked for gross correctness only (overall gradient error 4e-2 / 1.5e-1), the exact arithmetic being pinned by f32."""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

import oracle
from oracle import am_ref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# name -> (n_feat, n_label, B, T, L, scale_mode, transdiag)
CASES = {
    "conv_glu_wsj": (40, 30, 2, 150, 12, "target_sz_sqrt", 5.0),
    "seq2seq_tds_ctc": (80, 2000, 2, 160, 6, "none", 0.0),
    "conv_glu_librispeech": (40, 30, 2, 48, 10, "target_sz_sqrt", 4.0),
    "streaming_tds_ctc": (80, 2000, 2, 160, 6, "none", 0.0),
}
COND_TOL = 2e-4  # backward-error bound of the scalar LayerNorm gradients in the fp32-accurate mode (see run_case; the fp32 accumulation of the 3xTF32 GEMMs loses ~K * 1e-8)
TOL = {"f32": dict(emis=2e-4, loss=2e-4, overall=1e-2, per_param=5e-2),
       "tf32": dict(emis=2e-2, loss=2e-2, overall=4e-2, per_param=None),
       "bf16": dict(emis=6e-2, loss=6e-2, overall=1.5e-1, per_param=None)}


def run_case(name, precision):
    from wav2letter_b200 import archs, capi
    from wav2letter_b200.trainer import Trainer

    gen, crit, _, _ = archs.BASELINE_ARCHS[name]
    F, N, B, T, L, mode, transdiag = CASES[name]
    arch = am_ref.zero_dropout(gen())
    tr = Trainer(arch, F, N, crit, mode, transdiag=transdiag, lr=0.0, lrcrit=0.0, maxgradnorm=0.0, precision=precision)
    rng = np.random.default_rng(sum(name.encode()))
    feat = torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32)).cuda()
    hi = N - 1 if crit == "ctc" else N
    y = rng.integers(0, hi, (B, L)).astype(np.int32)
    y[1, L - 2:] = -1
    tgt = torch.from_numpy(y).cuda()
    flat = tr.get_flat(0, 0).clone()
    layout = tr.layout(0)
    emis = tr.forward(feat).clone()  # [B,T',N]
    loss = tr.step(feat, tgt, True, float(B)).clone()
    grads = tr.get_flat(0, 1).double()
    assert tr.skipped_steps() == 0
    torch.cuda.synchronize()
    # float64 reference of the same arch from the same parameters
    ref = am_ref.RefNet(arch, F, N, flat, layout)
    e64 = ref.forward(feat)
    assert tuple(e64.shape) == tuple(emis.shape), (e64.shape, emis.shape)
    e_np = e64.detach().float().cpu().numpy()
    if crit == "ctc":
        ol, ode = oracle.ctc(e_np, y, mode)
    else:
        trans = tr.get_flat(1, 0).cpu().numpy().reshape(N, N)
        ol, ode, _ = oracle.asg(e_np, y, trans, mode)
    e64.backward(torch.from_numpy(ode).to(e64.device).double())
    g64 = ref.grads_flat(layout, flat.numel())
    # what stock fp32 torch (TF32 off) makes of the same graph: scalar LayerNorm gains / biases are sums with heavy
    # cancellation (a shift of a tensor that is re-normalised right after), their fp32 noise floor is far above 1e-3
    t32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        ref32 = am_ref.RefNet(arch, F, N, flat, layout, dtype=torch.float32)
        e32 = ref32.forward(feat)
        e32.backward(torch.from_numpy(ode).to(e32.device))
        g32 = ref32.grads_flat(layout, flat.numel()).double()
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = t32
    emis_err = float((emis.double() - e64.detach()).abs().max() / e64.detach().abs().max())
    loss_err = float(np.abs(loss.cpu().numpy() - ol).max() / max(1e-6, np.abs(ol).max()))
    gmax = float(g64.abs().max())
    overall = float((grads - g64).abs().max() / gmax)
    per, excess, cond_worst = [], 0.0, 0.0
    for i, (o, n, dims) in enumerate(layout):
        own = float(g64[o:o + n].abs().max())
        err = float((grads[o:o + n] - g64[o:o + n]).abs().max())
        # per-parameter metric: relative L2 error (floor: a parameter whose whole gradient is below 1e-3 of the net's largest
        # entry is measured against that floor).  L2, not max-abs: at these reduced sizes a Linear sees only B*T' = 40 rows, so
        # ONE ReLU whose pre-activation changes sign between two correct fp32 evaluations (|pre| < 1e-5) moves single entries
        # of the following weight gradient by percents of the parameter's scale — a property of the kink, not an error
        l2 = float((grads[o:o + n] - g64[o:o + n]).norm())
        l2ref = max(float(g64[o:o + n].norm()), 1e-2 * gmax * (n ** 0.5))
        l2_32 = float((g32[o:o + n] - g64[o:o + n]).norm())
        denom = max(own, 1e-3 * gmax)
        per.append((l2 / l2ref, i, dims, own / gmax, l2_32 / l2ref, err / denom))
        if n == 1 and i in ref.cond:
            # scalar LayerNorm gain / bias: the gradient is ONE sum over every activation of the layer, with heavy
            # cancellation (a constant shift of a tensor that the next LayerNorm removes again) — its value can sit orders of
            # magnitude below the sum of the absolute contributions, so a relative criterion on the VALUE measures the
            # conditioning of the sum, not the kernels.  Backward-error bound instead: |error| <= COND_TOL * sum |contribution|
            cond_worst = max(cond_worst, err / max(ref.cond[i], 1e-30))
            continue
        # the f32 criterion: relative L2 error within 5e-2, or within 8x of stock fp32 torch's own error on that parameter
        excess = max(excess, l2 / max(5e-2 * l2ref, 8.0 * l2_32))
    per.sort(reverse=True)
    rec = {"arch": name, "precision": precision, "emis_err": emis_err, "loss_err": loss_err, "grad_overall": overall,
           "grad_worst_param": per[0][0], "worst_param_index": per[0][1], "worst_param_dims": list(per[0][2]),
           "worst5": [{"rel": round(q[0], 6), "index": q[1], "dims": list(q[2]), "own_over_gmax": round(q[3], 6), "torch_fp32_rel": round(q[4], 6), "max_abs_rel": round(q[5], 6)} for q in per[:5]],
           "f32_criterion_excess": excess, "scalar_ln_backward_error": cond_worst, "torch_fp32_overall": float((g32 - g64).abs().max() / gmax),
           "params": len(layout), "n_param_elements": int(flat.numel()), "loss": [float(v) for v in loss.cpu().numpy()]}
    with open(os.path.join(tempfile.gettempdir(), "w2l_arch_parity.jsonl"), "a") as f:
        f.write(json.dumps(rec) + "\n")
    tr.close()
    capi.set_precision("tf32")
    return rec


@pytest.mark.parametrize("name", sorted(CASES))
def test_arch_file_parity_fp32_accurate(name):
    rec = run_case(name, "f32")
    t = TOL["f32"]
    assert np.isfinite(rec["loss"]).all()
    assert rec["emis_err"] <= t["emis"], rec
    assert rec["loss_err"] <= t["loss"], rec
    # overall: within 1e-2 of the largest gradient entry, or 8x stock fp32 torch's own overall error
    assert rec["grad_overall"] <= max(t["overall"], 8 * rec["torch_fp32_overall"]), rec
    # every parameter: relative L2 error within 5e-2 (floor 1e-2 of the largest entry), or within 8x of stock fp32 torch's error
    assert rec["f32_criterion_excess"] <= 1.0, rec
    # scalar LayerNorm parameters: backward error (|error| / sum of absolute contributions) at the fp32 level
    assert rec["scalar_ln_backward_error"] <= COND_TOL, rec


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_arch_file_reduced_precision_modes(name, precision):
    rec = run_case(name, precision)
    t = TOL[precision]
    assert np.isfinite(rec["loss"]).all()
    assert rec["emis_err"] <= t["emis"], rec
    assert rec["loss_err"] <= t["loss"], rec
    assert rec["grad_overall"] <= t["overall"], rec


def test_tds_block_reference_golden():
    """The reference's own whole-TDS-block known answer (inference/module/test/TDSBlockTest.cpp:27-188, tolerance 1e-2):
    conv k=3 (pad 1/1) over 5 groups x 2 channels, per-frame LayerNorm, two Linear layers — fed through
    fl::TDSBlock(c=2, k=3, w=5, rPad=1, lnIncludeTime=0) of the CUDA path."""
    from wav2letter_b200.trainer import Trainer

    g = np.load(os.path.join(ROOT, "tests", "golden", "tds_block_golden.npz"))
    T, W, C, K = int(g["T"]), int(g["W"]), int(g["C"]), int(g["K"])
    nf = W * C
    arch = f"V -1 NFEAT 1 0\nV 0 {W} {C} 0\nTDS {C} {K} {W} 0 0 1 0\n"
    # the reference's inference layout is [T][w][c] (feature w*C + c); the internal one is [T][c][w] (feature c*W + w)
    perm = np.array([(f % W) * C + f // W for f in range(nf)])  # internal feature f -> reference feature
    x = g["in"].reshape(T, nf)[:, perm]                       # [T][internal feature]
    feat = torch.from_numpy(np.ascontiguousarray(x.T)[None, None]).float().cuda()  # [B=1,1,F,T]
    cw = g["conv_weights"].reshape(C, K, C).transpose(0, 2, 1)  # [cout][kw][cin] -> [cout][cin][kw]
    W1 = g["lin1_weights"].reshape(nf, nf)  # reference W[i*nOut + o]
    W2 = g["lin2_weights"].reshape(nf, nf)
    lin = lambda Wr: np.ascontiguousarray(Wr[perm][:, perm].T)  # -> memory [out][in] in internal feature order  # noqa: E731
    for precision in ("f32", "tf32", "bf16"):
        tr = Trainer(arch, nf, nf, "ctc", "none", precision=precision)
        parts = [cw.reshape(-1), g["conv_bias"], g["ln1_weights"], g["ln1_bias"], lin(W1).reshape(-1), g["lin1_bias"][perm],
                 lin(W2).reshape(-1), g["lin2_bias"][perm], g["ln2_weights"], g["ln2_bias"]]
        layout = tr.layout(0)
        assert [n for _, n, _ in layout] == [p.size for p in parts]
        flat = torch.zeros(tr.num_params(0))
        for (o, n, _), p in zip(layout, parts):
            flat[o:o + n] = torch.from_numpy(np.asarray(p, dtype=np.float32).reshape(-1))
        tr.set_flat(flat.cuda())
        out = tr.forward(feat).cpu().numpy().reshape(T, nf)  # [T][internal feature]
        exp = g["expectedOutput"].reshape(T, nf)[:, perm]
        err = float(np.abs(out - exp).max())
        tol = 1e-2 if precision != "bf16" else 5e-2
        assert err <= tol, (precision, err)
        tr.close()


def test_linseg_criterion_is_asg_on_the_stretched_target_and_trains():
    """LinSegCriterion (Train.cpp:589-617, --linseg warm start :1867-1883): loss = FCC - FAC on the linearly stretched
    target (ASG's signs), and one SGD step on it lowers the loss."""
    from wav2letter_b200.trainer import Trainer

    F, N, B, T, L = 40, 30, 3, 64, 7
    arch = "V -1 1 NFEAT 0\nWN 3 C NFEAT 60 5 1 -1\nGLU 2\nRO 2 0 3 1\nWN 0 L 30 NLABEL\n"
    rng = np.random.default_rng(5)
    feat = torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32)).cuda()
    y = rng.integers(0, N, (B, L)).astype(np.int32)
    y[2, 4:] = -1
    tgt = torch.from_numpy(y).cuda()
    tr = Trainer(arch, F, N, "linseg", "target_sz_sqrt", transdiag=2.0, lr=0.2, lrcrit=0.01, precision="f32")
    emis = tr.forward(feat).cpu().numpy()
    trans = tr.get_flat(1, 0).cpu().numpy().reshape(N, N)
    loss0 = tr.step(feat, tgt, True, float(B)).cpu().numpy()
    st = oracle.linseg_target(y, emis.shape[1])
    ol, _, odt = oracle.asg(emis, st, trans, "target_sz_sqrt")
    assert np.abs(loss0 - ol).max() <= 2e-4 * np.abs(ol).max(), (loss0, ol)
    assert (loss0 >= -1e-4).all()  # FCC >= FAC
    dtr = tr.get_flat(1, 1).cpu().numpy().reshape(N, N)
    assert np.abs(dtr - odt).max() <= 1e-3 * max(1e-6, np.abs(odt).max())
    for _ in range(3):
        loss1 = tr.step(feat, tgt, True, float(B)).cpu().numpy()
    assert loss1.sum() < loss0.sum(), (loss0, loss1)
    tr.close()
