"""slimIPL on the GPU (recipes/slimIPL/src/Train.cpp:396-404, 1362-1415, 1663-1673, 1823-1831):

- w2l_soft_label_loss against the float64 model of tests/slimipl_reference.py, bit-stable across runs, exactly 0 gradient
  for identical teacher and student rows;
- the teacher's EMA against the float32 model, bit for bit, across skipped updates and mixed-precision retries;
- the teacher's forward and viterbiPath against the pieces they are made of;
- the soft step against oracle/am_ref.py's float64 graph;
- hard and soft pseudo-labels end to end on an overfitted model, and checkpoints with a teacher."""
import struct

import numpy as np
import pytest
import torch

import slimipl_reference as ref
from oracle import am_ref

pytestmark = pytest.mark.gpu

F = 16
# a small TDS + CTC model without dropout (train- and eval-mode forwards are the same computation)
TDS_ARCH = """V -1 NFEAT 1 0
C2 1 4 5 1 1 1 -1 -1
R
TDS 4 5 16 0.0
V 0 64 1 0
RO 1 0 3 2
L 64 NLABEL
"""
# Soft-loss errors against float64, measured on an H100 80GB HBM3: at most 2.1e-7 relative on the loss and 3.0e-7 on the
# gradient (absolute, in units of scale / rows, i.e. on softmax(z) - p).  The bounds keep a margin of about 10x.
LOSS_TOL, GRAD_TOL = 2e-6, 3e-6


def _trainer(criterion="ctc", N=12, lr=0.05, momentum=0.5, precision="f32", arch=TDS_ARCH, maxgradnorm=0.0):
    from wav2letter_b200.trainer import Trainer

    return Trainer(arch, F, N, criterion, "none", transdiag=1.0, lr=lr, lrcrit=0.01 if criterion != "ctc" else 0.0, momentum=momentum,
                   maxgradnorm=maxgradnorm, precision=precision)


def _batch(rng, N, B=3, T=60, L=6, bad=False):
    feat = torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32)).cuda()
    y = rng.integers(0, N - 1, (B, L)).astype(np.int32)  # ctc: blank = N - 1
    y[1, L - 2:] = -1
    if bad:
        y[2, 1] = N  # not a token: that utterance's loss is NaN and the guard skips the update
    return feat, torch.from_numpy(y).cuda()


# ---- the soft-label loss kernel --------------------------------------------------------------------------------------
def _logits(rng, rows, N, offset, scale=3.0):
    buf = torch.empty(rows * N + offset, dtype=torch.float32, device="cuda")
    v = buf[offset:].view(rows, N)
    v.copy_(torch.from_numpy((rng.standard_normal((rows, N)) * scale).astype(np.float32)))
    return v


@pytest.mark.parametrize("peak", [1.0, 50.0])
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("rows", [1, 7, 2400])
@pytest.mark.parametrize("N", [29, 1000, 1001, 10000])
def test_soft_loss_kernel_against_float64(N, rows, offset, peak):
    from wav2letter_b200 import capi

    rng = np.random.default_rng(N * 7 + rows + offset)
    z = _logits(rng, rows, N, offset)
    t = _logits(rng, rows, N, offset, scale=peak)
    scale = 0.75
    dbuf = torch.empty(rows * N + offset, dtype=torch.float32, device="cuda")
    d_out = dbuf[offset:].view(rows, N)
    loss, d = capi.soft_label_loss(z, t, scale, d_student=d_out)
    torch.cuda.synchronize()
    # float64 reference on the device (the NumPy model of slimipl_reference, restated in torch for speed at 24M elements)
    z64, t64 = z.double(), t.double()
    p = torch.softmax(t64, -1)
    lq = torch.log_softmax(z64, -1)
    l64 = -scale / rows * float((p * lq).sum())
    d64 = scale / rows * (lq.exp() - p)
    if rows * N <= 100000:  # the NumPy model agrees with the torch restatement
        lm, dm = ref.soft_label_loss(z.cpu().numpy(), t.cpu().numpy(), scale)
        assert abs(lm - l64) <= 1e-12 * abs(l64) and np.abs(dm - d64.cpu().numpy()).max() <= 1e-12 * scale / rows
    loss_err = abs(float(loss) - l64) / max(abs(l64), 1e-30)
    grad_err = float((d.double() - d64).abs().max()) / (scale / rows)
    print(f"soft_loss N={N} rows={rows} offset={offset} peak={peak}: loss rel {loss_err:.3e}, grad {grad_err:.3e}")
    assert loss_err <= LOSS_TOL and grad_err <= GRAD_TOL, (loss_err, grad_err)
    # two runs give the same bits
    loss2, d2 = capi.soft_label_loss(z, t, scale)
    assert torch.equal(loss, loss2) and torch.equal(d, d2)
    # loss only: the same loss
    loss3, none = capi.soft_label_loss(z, t, scale, need_grad=False)
    assert none is None and torch.equal(loss, loss3)
    # identical teacher and student rows (the same buffer, and a copy): the gradient is exactly 0
    for same in (z, z.clone()):
        _, dz = capi.soft_label_loss(z, same, scale)
        assert int(torch.count_nonzero(dz)) == 0


def test_soft_loss_kernel_rejects_bad_arguments():
    from wav2letter_b200 import W2LError, capi

    z = torch.zeros((4, 10), device="cuda")
    with pytest.raises(ValueError):
        capi.soft_label_loss(z, torch.zeros((4, 11), device="cuda"))
    with pytest.raises(W2LError):
        capi.soft_label_loss(z, z, float("nan"))


# ---- the EMA kernel --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,offset", [(1, 0), (4099, 0), (1 << 20, 0), (1 << 20, 1), (4096, 3)])
@pytest.mark.parametrize("decay", [0.0, 0.9, 0.999, 1.0])
def test_ema_kernel_is_the_float32_model(n, offset, decay):
    from wav2letter_b200 import capi

    rng = np.random.default_rng(n + offset)
    e0 = rng.standard_normal(n).astype(np.float32)
    p = rng.standard_normal(n).astype(np.float32)
    eb = torch.empty(n + offset, dtype=torch.float32, device="cuda")
    pb = torch.empty(n + offset, dtype=torch.float32, device="cuda")
    e, pd = eb[offset:], pb[offset:]
    e.copy_(torch.from_numpy(e0))
    pd.copy_(torch.from_numpy(p))
    capi.ema_update(e, pd, decay)
    want = ref.ema_update(e0, p, decay)
    assert np.array_equal(e.cpu().numpy().view(np.int32), want.view(np.int32))


# ---- the teacher in the trainer --------------------------------------------------------------------------------------
def _np(x):
    return x.cpu().numpy()


def test_teacher_follows_the_float32_model_across_skipped_updates():
    N, decay = 12, 0.9
    rng = np.random.default_rng(5)
    tr = _trainer(N=N)
    assert tr.ema() is None and tr.num_params(2) == tr.num_params(0)
    assert torch.equal(tr.get_flat(2), tr.get_flat(0))  # without a teacher, the teacher is the network
    tr.set_ema(decay)
    assert tr.ema() == decay and "EMA teacher" in tr.describe()
    e = _np(tr.get_flat(2))
    assert np.array_equal(e, _np(tr.get_flat(0)))
    batches = [_batch(rng, N) for _ in range(3)] + [_batch(rng, N, bad=True)] + [_batch(rng, N) for _ in range(2)]
    skipped = 0
    for k, (feat, tgt) in enumerate(batches):
        before = _np(tr.get_flat(0))
        tr.step(feat, tgt, total_batch=3.0)
        p = _np(tr.get_flat(0))
        if k == 3:  # the guard skipped this update: the network did not move, the teacher still did
            skipped += 1
            assert np.array_equal(p, before)
        e = ref.ema_update(e, p, decay)
        assert tr.skipped_steps() == skipped
        assert np.array_equal(_np(tr.get_flat(2)).view(np.int32), e.view(np.int32)), k
    # eval steps leave the teacher alone
    tr.step(*batches[0], train=False)
    assert np.array_equal(_np(tr.get_flat(2)), e)
    # forward of the teacher = a trainer whose network holds the teacher's values
    other = _trainer(N=N)
    other.set_flat(tr.get_flat(2), 0)
    feat = batches[0][0]
    assert torch.equal(tr.forward(feat, teacher=True), other.forward(feat))
    assert not torch.equal(tr.forward(feat, teacher=True), tr.forward(feat))
    # set_flat(which=2) writes the teacher; dropping it makes the teacher the network again
    tr.set_flat(tr.get_flat(0), 2)
    assert torch.equal(tr.forward(feat, teacher=True), tr.forward(feat))
    tr.set_ema(None)
    assert tr.ema() is None and "EMA teacher" not in tr.describe()
    tr.close()
    other.close()


def test_teacher_is_updated_once_per_batch_under_mixed_precision_retries():
    N, decay = 12, 0.75
    rng = np.random.default_rng(6)
    tr = _trainer(N=N, precision="fp16")
    tr.set_ema(decay)
    e = _np(tr.get_flat(2))
    tr.set_amp(True, initial_scale=2.0 ** 40)
    for k in range(2):
        feat, tgt = _batch(rng, N)
        retries = tr.amp_state()[2]
        tr.step(feat, tgt)
        if k == 0:
            assert tr.amp_state()[2] > retries  # fp16 gradients at 2^40 times the loss overflow: the batch ran again
        e = ref.ema_update(e, _np(tr.get_flat(0)), decay)
        assert np.array_equal(_np(tr.get_flat(2)).view(np.int32), e.view(np.int32)), k
    assert tr.skipped_steps() == 0
    tr.close()


@pytest.mark.parametrize("decay", [0.0, 1.0])
def test_teacher_at_decay_0_is_the_network_and_at_decay_1_stays(decay):
    N = 12
    rng = np.random.default_rng(7)
    tr = _trainer(N=N)
    tr.set_ema(decay)
    e0 = tr.get_flat(2).clone()
    for _ in range(3):
        tr.step(*_batch(rng, N), total_batch=3.0)
    assert not torch.equal(tr.get_flat(0), e0)
    assert torch.equal(tr.get_flat(2), tr.get_flat(0) if decay == 0.0 else e0)
    tr.close()


def test_set_ema_rejects_bad_decays():
    from wav2letter_b200 import W2LError

    tr = _trainer()
    for d in (-0.1, 1.5, float("nan")):
        with pytest.raises(W2LError):
            tr.set_ema(d)
    assert tr.ema() is None
    with pytest.raises(W2LError):
        tr.get_flat(2, 1)  # the teacher has no gradients
    tr.close()


# ---- viterbiPath -----------------------------------------------------------------------------------------------------
def test_viterbi_path_ctc_is_the_argmax_of_the_forward():
    from wav2letter_b200 import W2LError, argmax_path

    N = 12
    rng = np.random.default_rng(8)
    tr = _trainer(N=N)
    tr.set_ema(0.5)
    for _ in range(2):
        tr.step(*_batch(rng, N), total_batch=3.0)
    feat, _ = _batch(rng, N)
    for teacher in (False, True):
        assert torch.equal(tr.viterbi_path(feat, teacher=teacher), argmax_path(tr.forward(feat, teacher=teacher)))
    with pytest.raises(W2LError):
        tr.viterbi_path(feat, input_sizes=[60, 50, 40])  # sizes are the seq2seq criterion's
    tr.close()


def test_viterbi_path_asg_is_the_fcc_viterbi_of_the_forward():
    from wav2letter_b200 import fcc_viterbi

    N = 10
    rng = np.random.default_rng(9)
    tr = _trainer("asg", N=N)
    tr.set_flat(torch.from_numpy(rng.standard_normal(N * N).astype(np.float32)).cuda(), 1)
    tr.set_ema(0.5)
    tr.step(*_batch(rng, N), total_batch=3.0)
    feat, _ = _batch(rng, N)
    trans = tr.get_flat(1).view(N, N)
    for teacher in (False, True):
        assert torch.equal(tr.viterbi_path(feat, teacher=teacher), fcc_viterbi(tr.forward(feat, teacher=teacher), trans))
    tr.close()


def test_viterbi_path_seq2seq_is_the_greedy_decode():
    import test_gpu_seq2seq as s2s

    rng = np.random.default_rng(10)
    tr = s2s.make_trainer(32, 10, maxlen=12, lr=0.05, lrcrit=0.05)
    B, T = 3, 40
    feat = s2s.features(rng, B, T)
    tgt = torch.from_numpy(s2s.targets(rng, B, 6, 10)).cuda()
    for _ in range(3):
        tr.step(feat, tgt)
    tokens, _ = tr.decode(feat)
    path = tr.viterbi_path(feat)
    assert path.shape == tokens.shape and torch.equal(path, tokens)
    sizes = [40, 30, 22]
    assert torch.equal(tr.viterbi_path(feat, input_sizes=sizes), tr.decode(feat, input_sizes=sizes)[0])
    tr.close()


# ---- the soft step ---------------------------------------------------------------------------------------------------
COND_TOL = 2e-4  # tests/test_gpu_archs.py: backward error of the scalar LayerNorm gradients in f32


def test_soft_step_against_float64():
    """one f32 soft step with lr = 0: the loss and every parameter gradient against am_ref's float64 graph with the loss
    soft_scale * -mean_{t,b} sum_c softmax(teacher) logSoftmax(output), by test_gpu_archs.py's per-parameter criterion"""
    N, B, T, scale = 30, 2, 70, 0.6
    rng = np.random.default_rng(11)
    tr = _trainer(N=N, lr=0.0, momentum=0.0)
    feat = torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32)).cuda()
    flat, layout = tr.get_flat(0, 0).clone(), tr.layout(0)
    Tp = tr.forward(feat).shape[1]
    teacher = torch.from_numpy((rng.standard_normal((B, Tp, N)) * 4).astype(np.float32)).cuda()
    loss = tr.step_soft(feat, teacher, soft_scale=scale, total_batch=1.0)
    grads = tr.get_flat(0, 1).double()
    assert loss.shape == (1,) and tr.skipped_steps() == 0
    assert torch.equal(tr.get_flat(0), flat)  # lr = 0

    def ref_grads(dtype):
        net = am_ref.RefNet(TDS_ARCH, F, N, flat, layout, dtype=dtype)
        out = net.forward(feat)
        l = scale * -(torch.softmax(teacher.to(dtype), -1) * torch.log_softmax(out, -1)).sum(-1).mean()
        l.backward()
        return float(l.detach()), net.grads_flat(layout, flat.numel()).double(), net

    t32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        l64, g64, net64 = ref_grads(torch.float64)
        _, g32, _ = ref_grads(torch.float32)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = t32
    assert abs(float(loss) - l64) <= 2e-4 * abs(l64), (float(loss), l64)
    gmax = float(g64.abs().max())
    for i, (o, n, dims) in enumerate(layout):
        err = float((grads[o:o + n] - g64[o:o + n]).abs().max())
        if n == 1 and i in net64.cond:
            assert err <= COND_TOL * max(net64.cond[i], 1e-30), (i, dims, err)
            continue
        l2 = float((grads[o:o + n] - g64[o:o + n]).norm())
        l2ref = max(float(g64[o:o + n].norm()), 1e-2 * gmax * (n ** 0.5))
        l2_32 = float((g32[o:o + n] - g64[o:o + n]).norm())
        assert l2 <= max(5e-2 * l2ref, 8.0 * l2_32), (i, dims, l2 / l2ref)
    tr.close()


def test_soft_step_against_its_own_output_changes_nothing():
    """no dropout or SAUG: the train-mode forward has the eval-mode forward's bits, so with teacher_logits = forward() every
    gradient is exactly 0 and SGD (momentum 0) leaves every parameter as it was"""
    from wav2letter_b200 import ctc_forward_backward

    N = 12
    rng = np.random.default_rng(12)
    tr = _trainer(N=N, lr=0.0, momentum=0.0)
    feat, tgt = _batch(rng, N)
    # the premise: the CTC loss of a training step (train-mode forward, lr 0) has the bits of the same CTC kernel's loss on
    # the eval-mode forward
    want, _ = ctc_forward_backward(tr.forward(feat), tgt, "none")
    assert torch.equal(tr.step(feat, tgt, total_batch=3.0), want)
    tr.set_lr(0.5, 0.5)
    before = tr.get_flat(0).clone()
    loss = tr.step_soft(feat, tr.forward(feat), soft_scale=1.0)
    assert torch.isfinite(loss).all() and float(loss) > 0.0  # the teacher's entropy
    assert int(torch.count_nonzero(tr.get_flat(0, 1))) == 0
    assert torch.equal(tr.get_flat(0), before)
    tr.close()


def test_soft_step_rejects_a_teacher_of_another_shape():
    from wav2letter_b200 import W2LError

    N = 12
    rng = np.random.default_rng(13)
    tr = _trainer(N=N)
    feat, _ = _batch(rng, N)
    out = tr.forward(feat)
    with pytest.raises(W2LError):
        tr.step_soft(feat, out[:, 1:].contiguous())
    with pytest.raises(ValueError):
        tr.step_soft(feat, torch.zeros((out.shape[0], out.shape[1], N + 1), device="cuda"))
    tr.close()


# ---- end to end ------------------------------------------------------------------------------------------------------
LETTERS = "|\n'\n" + "\n".join("abcdefghijklmnopqrstuvwxyz") + "\n"
TRANSCRIPTS = ["hi yo", "abc", "bad cab"]


def _spoken(rng, text, transcripts, T=96, noise=0.1):
    """features that spell each transcript: every token 4 frames of its own code, 4 frames of silence between tokens"""
    code = np.random.default_rng(99).standard_normal((text.num_classes, F)).astype(np.float32)
    feat = (rng.standard_normal((len(transcripts), 1, F, T)) * noise).astype(np.float32)
    for b, s in enumerate(transcripts):
        for k, tok in enumerate(text.encode(s)):
            feat[b, 0, :, 4 + 8 * k:8 + 8 * k] += code[tok][:, None]
    return torch.from_numpy(feat).cuda()


def test_pseudo_labels_and_a_naive_slimipl_loop():
    from wav2letter_b200.slimipl import pl_strings, pseudo_labels, soft_targets
    from wav2letter_b200.text import TextPipeline

    text = TextPipeline(LETTERS, "", "ctc", 0, "", False, "|")
    N = text.num_classes
    rng = np.random.default_rng(14)
    tr = _trainer(N=N, lr=0.05, momentum=0.9, maxgradnorm=1.0)
    feat = _spoken(rng, text, TRANSCRIPTS)
    tgt = torch.from_numpy(text.encode_batch(TRANSCRIPTS)).cuda()
    for i in range(2000):
        tr.step(feat, tgt, total_batch=3.0)
        if i % 50 == 49 and pl_strings(text, tr.viterbi_path(feat).cpu().numpy()) == TRANSCRIPTS:
            break
    assert tr.skipped_steps() == 0
    tr.set_ema(0.999)
    targets, sizes, strings = pseudo_labels(tr, text, feat)
    assert strings == TRANSCRIPTS
    assert torch.equal(targets, tgt)
    assert sizes.tolist() == [len(text.encode(s)) for s in TRANSCRIPTS]
    # one supervised step, then one step on an unlabelled batch (new noise) with its hard or soft PLs
    for soft in (False, True):
        for _ in range(3):
            assert torch.isfinite(tr.step(feat, tgt, total_batch=3.0)).all()
            unl = _spoken(rng, text, TRANSCRIPTS)
            if soft:
                loss = tr.step_soft(unl, soft_targets(tr, unl), soft_scale=1.0)
            else:
                pl, _, _ = pseudo_labels(tr, text, unl)
                loss = tr.step(unl, pl, total_batch=3.0)
            assert torch.isfinite(loss).all()
    assert tr.skipped_steps() == 0
    tr.close()


# ---- checkpoints -----------------------------------------------------------------------------------------------------
def _version(path):
    with open(path, "rb") as f:
        return struct.unpack("<8sI", f.read(12))[1]


def test_checkpoints_with_and_without_a_teacher(tmp_path):
    from wav2letter_b200.trainer import Trainer

    N = 12
    rng = np.random.default_rng(15)
    tr = _trainer(N=N)
    tr.step(*_batch(rng, N), total_batch=3.0)
    v2, v2b = str(tmp_path / "v2.bin"), str(tmp_path / "v2b.bin")
    tr.save(v2)
    assert _version(v2) == 2
    # without a teacher the file is what a trainer that never had one writes, byte for byte
    tr.set_ema(0.95)
    tr.set_ema(None)
    tr.save(v2b)
    with open(v2, "rb") as f:
        b2 = f.read()
    with open(v2b, "rb") as f:
        assert f.read() == b2
    # with a teacher: version 4 = the version 2 bytes of the same trainer, then f64 decay and the teacher's arena
    tr.set_ema(0.95)
    tr.step(*_batch(rng, N), total_batch=3.0)
    vt = str(tmp_path / "teacher.bin")
    tr.save(vt)
    ema = tr.get_flat(2).clone()
    tr.set_ema(None)
    tr.save(v2b)
    with open(v2b, "rb") as f:
        b2 = f.read()
    with open(vt, "rb") as f:
        bt = f.read()
    assert _version(vt) == 4 and bt[:8] == b2[:8] and bt[12:len(b2)] == b2[12:]
    n = tr.num_params(2)
    assert len(bt) == len(b2) + 8 + 8 + 4 * n
    assert struct.unpack("<d", bt[len(b2):len(b2) + 8])[0] == 0.95
    assert np.array_equal(np.frombuffer(bt[len(b2) + 16:], np.float32), ema.cpu().numpy())
    # a version 4 file restores the teacher, and runs continue bit for bit
    a = Trainer.load(vt)
    b = Trainer.load(vt)
    assert a.ema() == 0.95 and torch.equal(a.get_flat(2), ema)
    feat, tgt = _batch(rng, N)
    a.step(feat, tgt, total_batch=3.0)
    b.step(feat, tgt, total_batch=3.0)
    assert torch.equal(a.get_flat(2), b.get_flat(2)) and not torch.equal(a.get_flat(2), ema)
    # version 2 files load without a teacher
    c = Trainer.load(v2)
    assert c.ema() is None and torch.equal(c.get_flat(2), c.get_flat(0))
    for t in (tr, a, b, c):
        t.close()
