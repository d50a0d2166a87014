"""The Seq2Seq criterion (--criterion=seq2seq) on the GPU against the float64 oracle (oracle/seq2seq_ref.py): loss and every
criterion and encoder parameter gradient through the trainer, the random draws reproduced by tests/seq2seq_reference.py,
batch invariance, launch counts, greedy decode, an overfitting run, mixed precision, checkpoints and errors."""
import os
import tempfile

import numpy as np
import pytest
import torch

import seq2seq_reference as S
from oracle import am_ref
from oracle import seq2seq_ref as ref

pytestmark = pytest.mark.gpu

F = 16  # filterbanks of the test encoder: one strided C2 (T' = T / 2), then `L 2F 2H`


def encoder_arch(H, width=None):
    return f"V -1 NFEAT 1 0\nC2 1 2 5 1 2 1 -1 -1\nR\nV 0 {2 * F} 1 0\nRO 1 0 3 2\nL {2 * F} {width or 2 * H}\n"


def make_trainer(H, N, maxlen=20, precision="f32", lr=0.0, lrcrit=0.0, momentum=0.0, maxgradnorm=0.0, width=None, **s2s):
    from wav2letter_b200.trainer import Trainer

    cfg = dict(hidden=H, eos=N - 2, pad=N - 1, maxdecoderoutputlen=maxlen, **s2s)
    return Trainer(encoder_arch(H, width), F, N, "seq2seq", lr=lr, lrcrit=lrcrit, momentum=momentum, maxgradnorm=maxgradnorm,
                   precision=precision, seq2seq=cfg)


def targets(rng, B, U, N, lengths=None):
    """tokens in [0, N-2), then eos, then pad"""
    y = np.full((B, U), N - 1, np.int32)
    for b in range(B):
        n = int(rng.integers(1, U)) if lengths is None else lengths[b]
        y[b, :n] = rng.integers(0, N - 2, n)
        y[b, n] = N - 2
    return y


def features(rng, B, T):
    return torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32)).cuda()


def max_rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


CASES = {
    # name: H, N, B, T, U, rounds, layers, dropout, labelsmooth, pct, window_std, train_with_window, train
    "small_r1s1": (32, 13, 3, 40, 7, 1, 1, 0.0, 0.0, 100, 0.0, False, True),
    "small_r1s1_window_ls": (32, 13, 3, 40, 7, 1, 1, 0.0, 0.05, 99, 3.0, True, True),
    "small_r2s3_dropout": (32, 13, 3, 40, 7, 2, 3, 0.1, 0.05, 99, 0.0, False, True),
    "small_r2s3_window_eval": (32, 13, 3, 40, 7, 2, 3, 0.1, 0.05, 99, 3.0, False, False),
    "recipe_r1s1": (512, 10002, 4, 300, 61, 1, 1, 0.0, 0.05, 99, 4.0, True, True),
    "recipe_r2s3": (512, 10002, 4, 300, 61, 2, 3, 0.1, 0.0, 100, 0.0, False, True),
    # --encoderdim=1024 (sota/2019 librivox tds_s2s): the backward stages dgh 8 rows at a time beside its 96 KB W_hh
    # slice; 18 utterances run the forward in chunks of 16 + 2 and the backward in 8 + 8 + 2
    "h1024_r1s2": (1024, 13, 18, 40, 7, 1, 2, 0.1, 0.05, 99, 3.0, True, True),
}


@pytest.mark.parametrize("name", list(CASES))
def test_parity_f32(name):
    H, N, B, T, U, R, L, p, ls, pct, wstd, tww, train = CASES[name]
    rng = np.random.default_rng(sum(name.encode()))
    tr = make_trainer(H, N, rounds=R, layers=L, dropout=p, labelsmooth=ls, pctteacherforcing=pct, window_std=wstd, train_with_window=tww)
    feat = features(rng, B, T)
    y = targets(rng, B, U, N)
    net_flat, crit_flat = tr.get_flat(0, 0).clone(), tr.get_flat(1, 0).clone()
    loss = tr.step(feat, torch.from_numpy(y).cuda(), train=train).cpu().numpy()
    torch.cuda.synchronize()
    enc = am_ref.RefNet(encoder_arch(H), F, N, net_flat, tr.layout(0), device="cpu")
    x = enc.forward(feat.cpu())
    params = ref.unflatten(crit_flat, tr.layout(1), N, H, R, L)
    if train:
        seed = tr.seq2seq_seed()
        tokens = S.substituted_tokens(seed, y, N, pct)
        masks = [S.dropout_scales(seed, k, (B, U, H), p) for k in range(R * L)] if p > 0 else None
        want = ref.loss(params, x, y, N - 1, tokens, R, L, wstd if tww else 0.0, ls, masks)
    else:
        want = ref.loss(params, x, y, N - 1, ref.teacher_tokens(y, N), R, L, wstd, 0.0)
    assert max_rel(loss, want.detach().numpy()) < 1e-4, (loss, want)
    if not train:
        return
    want.sum().backward()
    got_c = tr.get_flat(1, 1).double().cpu()
    for i, (po, (off, n, _)) in enumerate(zip(params, tr.layout(1))):
        g = po.grad.reshape(-1).numpy()
        assert max_rel(got_c[off:off + n].numpy(), g) < 2e-4, (name, "criterion parameter", i, max_rel(got_c[off:off + n].numpy(), g))
    got_n = tr.get_flat(0, 1).double().cpu()
    for i, (po, (off, n, _)) in enumerate(zip(enc.params, tr.layout(0))):
        g = po.grad.reshape(-1).numpy()
        assert max_rel(got_n[off:off + n].numpy(), g) < 2e-4, (name, "encoder parameter", i, max_rel(got_n[off:off + n].numpy(), g))


def test_substitution_is_reproduced():
    """at pctteacherforcing = 99 / 50 the decoder reads the substituted tokens the NumPy model predicts"""
    H, N, B, T, U = 32, 13, 4, 40, 30
    rng = np.random.default_rng(5)
    tr = make_trainer(H, N, pctteacherforcing=50)
    feat = features(rng, B, T)
    y = targets(rng, B, U, N, lengths=[U - 1] * B)
    net_flat, crit_flat = tr.get_flat(0, 0).clone(), tr.get_flat(1, 0).clone()
    loss = tr.step(feat, torch.from_numpy(y).cuda()).cpu().numpy()
    seed = tr.seq2seq_seed()
    tokens = S.substituted_tokens(seed, y, N, 50)
    assert (tokens[:, 1:] != ref.teacher_tokens(y, N).numpy()[:, 1:]).mean() > 0.2
    x = am_ref.RefNet(encoder_arch(H), F, N, net_flat, tr.layout(0), device="cpu").forward(feat.cpu())
    params = ref.unflatten(crit_flat, tr.layout(1), N, H)
    assert max_rel(loss, ref.loss(params, x, y, N - 1, tokens).detach().numpy()) < 1e-4


def test_batch_invariance():
    """without the window, each utterance's loss and gradient are those of a run with it alone, target trimmed"""
    H, N, B, T, U = 32, 13, 3, 40, 9
    rng = np.random.default_rng(11)
    tr = make_trainer(H, N)
    feat = features(rng, B, T)
    y = targets(rng, B, U, N, lengths=[2, 7, 4])
    loss = tr.step(feat, torch.from_numpy(y).cuda(), total_batch=1.0).cpu().numpy()
    gn, gc = tr.get_flat(0, 1).double().cpu(), tr.get_flat(1, 1).double().cpu()
    sn, sc = torch.zeros_like(gn), torch.zeros_like(gc)
    for b in range(B):
        n = int(np.argmax(y[b] == N - 2)) + 1
        lb = tr.step(feat[b:b + 1].contiguous(), torch.from_numpy(y[b:b + 1, :n].copy()).cuda(), total_batch=1.0).cpu().numpy()
        assert abs(lb[0] - loss[b]) <= 1e-5 * max(1.0, abs(loss[b])), (b, lb, loss)
        sn += tr.get_flat(0, 1).double().cpu()
        sc += tr.get_flat(1, 1).double().cpu()
    assert max_rel(gn.numpy(), sn.numpy()) < 1e-5
    assert max_rel(gc.numpy(), sc.numpy()) < 1e-5


def test_launch_count_independent_of_length():
    from wav2letter_b200 import capi

    H, N, B, T = 32, 13, 2, 40
    rng = np.random.default_rng(3)
    tr = make_trainer(H, N, rounds=2, layers=2)
    feat = features(rng, B, T)
    counts = {}
    for U in (20, 100):
        y = torch.from_numpy(targets(rng, B, U, N)).cuda()
        tr.step(feat, y)  # warm
        torch.cuda.synchronize()
        got = capi.trace(lambda: tr.step(feat, y))
        counts[U] = {k: v[0] for k, v in got.items() if "seq2seq" in k}
    assert counts[20] == counts[100], counts
    assert counts[20]["seq2seq_gru_fwd_kernel"] == 4 and counts[20]["seq2seq_gru_bwd_kernel"] == 4, counts[20]


def test_greedy_decode():
    H, N, B, T, maxlen = 32, 13, 4, 40, 12
    rng = np.random.default_rng(17)
    tr = make_trainer(H, N, maxlen=maxlen, rounds=2, layers=3)
    feat = features(rng, B, T)
    tokens, lengths = tr.decode(feat)
    tokens, lengths = tokens.cpu().numpy(), lengths.cpu().numpy()
    x = am_ref.RefNet(encoder_arch(H), F, N, tr.get_flat(0, 0), tr.layout(0), device="cpu").forward(feat.cpu())
    params = ref.unflatten(tr.get_flat(1, 0), tr.layout(1), N, H, 2, 3)
    for b, (want, gaps) in enumerate(ref.greedy(params, x.detach(), N - 2, maxlen, 2, 3)):
        got = list(tokens[b, :lengths[b]])
        for i, (g, w) in enumerate(zip(got, want)):
            if gaps[i] < 1e-3:
                break
            assert g == w, (b, i, got, want)
        else:
            assert len(got) == len(want) or min(gaps[:min(len(got), len(want)) + 1]) < 1e-3, (b, got, want)
        assert (tokens[b, lengths[b]:] == N - 1).all()
    # a batch decodes as its utterances alone
    for b in range(B):
        tb, lb = tr.decode(feat[b:b + 1].contiguous())
        assert int(lb[0]) == lengths[b] and (tb[0].cpu().numpy() == tokens[b]).all()
    # stops at eos (not emitted) and at the maximum length
    crit = tr.get_flat(1, 0).clone()
    bo = tr.layout(1)[-1][0]
    crit[bo + N - 2] = 1e4
    tr.set_flat(crit, 1)
    t2, l2 = tr.decode(feat)
    assert (l2.cpu().numpy() == 0).all() and (t2.cpu().numpy() == N - 1).all()
    crit[bo + N - 2] = -1e4
    crit[bo + 3] = 1e4
    tr.set_flat(crit, 1)
    t3, l3 = tr.decode(feat)
    assert (l3.cpu().numpy() == maxlen).all() and (t3.cpu().numpy() == 3).all()


def test_overfit_one_batch_and_decode():
    H, N, B, T, U = 64, 10, 2, 48, 6
    rng = np.random.default_rng(23)
    tr = make_trainer(H, N, maxlen=10, lr=0.05, lrcrit=0.5, momentum=0.9, maxgradnorm=5.0, window_std=4.0, train_with_window=True)
    feat = features(rng, B, T)
    y = targets(rng, B, U, N, lengths=[4, 5])
    tgt = torch.from_numpy(y).cuda()
    first = float(tr.step(feat, tgt).sum())
    assert tr.seq2seq_config()["window_set"] == 1
    for i in range(600):
        if i == 20:
            tr.clear_window()
            assert tr.seq2seq_config()["window_set"] == 0
        tr.step(feat, tgt)
        last = float(tr.step(feat, tgt, train=False).sum())
        if last < first / 10 and i > 50:
            break
    assert last < first / 10, (first, last)
    tokens, lengths = tr.decode(feat)
    for b, n in enumerate((4, 5)):
        assert int(lengths[b]) == n and (tokens[b, :n].cpu().numpy() == y[b, :n]).all(), (tokens, y)


def test_mixed_precision():
    H, N, B, T, U = 32, 13, 3, 40, 7
    rng = np.random.default_rng(29)
    feat = features(rng, B, T)
    tgt = torch.from_numpy(targets(rng, B, U, N)).cuda()
    tr = make_trainer(H, N, precision="fp16", lr=0.01, lrcrit=0.01)
    tr.set_amp(True)
    for _ in range(5):
        assert torch.isfinite(tr.step(feat, tgt)).all()
    scale, counter, retries = tr.amp_state()
    assert tr.skipped_steps() == 0 and retries == 0 and scale == 4096.0 + 2 * 5 and counter == 6
    a = make_trainer(H, N, precision="f32")
    b = make_trainer(H, N, precision="bf16")
    b.set_flat(a.get_flat(0, 0), 0)
    b.set_flat(a.get_flat(1, 0), 1)
    la, lb = a.step(feat, tgt, train=False).cpu().numpy(), b.step(feat, tgt, train=False).cpu().numpy()
    assert max_rel(lb, la) < 2e-2


def test_checkpoint_roundtrip():
    from wav2letter_b200.trainer import Trainer

    H, N, B, T, U = 32, 13, 2, 40, 7
    rng = np.random.default_rng(31)
    feat = features(rng, B, T)
    tgt = torch.from_numpy(targets(rng, B, U, N)).cuda()
    tr = make_trainer(H, N, lr=0.05, lrcrit=0.1, momentum=0.9, window_std=3.0, train_with_window=True)
    for _ in range(3):
        tr.step(feat, tgt)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "s2s.bin")
        tr.save(path)
        tr2 = Trainer.load(path)
    assert tr2.seq2seq_config() == tr.seq2seq_config() and tr2.output_width() == 2 * H
    l1, l2 = tr.step(feat, tgt), tr2.step(feat, tgt)
    assert torch.equal(l1, l2)
    for w in (0, 1):
        assert torch.equal(tr.get_flat(w, 0), tr2.get_flat(w, 0))


def test_errors():
    from wav2letter_b200 import W2LError

    H, N, B, T, U = 32, 13, 2, 40, 7
    rng = np.random.default_rng(37)
    feat = features(rng, B, T)
    y = targets(rng, B, U, N)
    with pytest.raises(W2LError, match="2 \\* encoderdim"):
        make_trainer(H, N, width=2 * H + 4).step(feat, torch.from_numpy(y).cuda())
    # a target value outside [0, N) is rejected on the device: that utterance's loss is NaN, the finite guard skips
    # the update, and the other utterance is untouched
    tr = make_trainer(H, N, lr=0.1, lrcrit=0.1)
    before = (tr.get_flat(0, 0).clone(), tr.get_flat(1, 0).clone())
    good = tr.step(feat, torch.from_numpy(y).cuda(), train=False).cpu().numpy()
    for v in (-1, N):
        bad = y.copy()
        bad[0, -1] = v
        loss = tr.step(feat, torch.from_numpy(bad).cuda()).cpu().numpy()
        assert np.isnan(loss[0]) and loss[1] == good[1], (v, loss, good)
    assert tr.skipped_steps() == 2
    assert torch.equal(tr.get_flat(0, 0), before[0]) and torch.equal(tr.get_flat(1, 0), before[1])
    with pytest.raises(W2LError, match="seq2seq"):
        tr.align(feat, torch.from_numpy(y).cuda())
    with tempfile.TemporaryDirectory() as d, pytest.raises(W2LError, match="seq2seq"):
        tr.export_streaming(d)
    with pytest.raises(W2LError, match="multiple of 32"):
        make_trainer(48, N)
    with pytest.raises(W2LError):
        make_trainer(H, N, rounds=0)
    assert tr.forward(feat).shape == (B, T // 2, 2 * H)
