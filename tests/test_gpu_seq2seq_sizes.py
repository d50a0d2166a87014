"""The Seq2Seq criterion on padded batches on the GPU: per-utterance encoder lengths and target sizes.

Through the trainer: f32 parity of the loss and every criterion and encoder gradient against float64 (oracle/am_ref.py's
encoder and tests/seq2seq_sizes_reference.py), full sizes against no sizes bit for bit, bf16 with loss scaling, the
in-band rejection of bad sizes, refusals and launch counts.  On a given encoder output (tests/seq2seq_sizes/
criterion_sized.cpp, compiled against fl_compat.h): each utterance of a padded batch against a run on its own frames
and target, bit for bit, and NaN padding that changes nothing, for the loss, the encoder gradient, the greedy decode and
the beam search."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import seq2seq_reference as S
import seq2seq_sizes_reference as SR
from oracle import am_ref
from oracle import seq2seq_ref as ref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = 16  # filterbanks of the test encoder: one strided C2 (T' = T / 2), then `L 2F 2H`


def encoder_arch(H):
    return f"V -1 NFEAT 1 0\nC2 1 2 5 1 2 1 -1 -1\nR\nV 0 {2 * F} 1 0\nRO 1 0 3 2\nL {2 * F} {2 * H}\n"


def make_trainer(H, N, maxlen=20, precision="f32", lr=0.0, lrcrit=0.0, **s2s):
    from wav2letter_b200.trainer import Trainer

    cfg = dict(hidden=H, eos=N - 2, pad=N - 1, maxdecoderoutputlen=maxlen, **s2s)
    return Trainer(encoder_arch(H), F, N, "seq2seq", lr=lr, lrcrit=lrcrit, precision=precision, seq2seq=cfg)


def targets(rng, B, U, N, lengths):
    """tokens in [0, N-2), then eos, then pad; returns (y, target sizes = tokens + eos)"""
    y = np.full((B, U), N - 1, np.int32)
    for b, n in enumerate(lengths):
        y[b, :n] = rng.integers(0, N - 2, n)
        y[b, n] = N - 2
    return y, [n + 1 for n in lengths]


def max_rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


CASES = {
    # name: H, N, B, T, U, rounds, layers, dropout, labelsmooth, pct, window_std, train_with_window, train
    "small_r1s1": (32, 13, 4, 40, 9, 1, 1, 0.0, 0.0, 100, 0.0, False, True),
    "small_r1s1_window_ls": (32, 13, 4, 40, 9, 1, 1, 0.0, 0.05, 99, 3.0, True, True),
    "small_r2s3_dropout": (32, 13, 4, 40, 9, 2, 3, 0.1, 0.05, 99, 0.0, False, True),
    "small_r2s3_window_eval": (32, 13, 4, 40, 9, 2, 3, 0.1, 0.05, 99, 3.0, False, False),
    "recipe_r1s1_window": (512, 10002, 16, 300, 61, 1, 1, 0.0, 0.05, 99, 4.0, True, True),
    "recipe_r2s3_dropout": (512, 10002, 16, 300, 61, 2, 3, 0.1, 0.0, 100, 0.0, False, True),
}


def spread(rng, B, T, U):
    """input frame counts from about 0.4 T to T (the longest is T) and token counts from about U / 3 to U - 1"""
    d = rng.integers(int(0.4 * T), T + 1, B)
    d[0], d[-1] = T, int(0.4 * T)
    n = rng.integers(max(1, U // 3), U, B)
    n[0], n[-1] = U - 1, max(1, U // 3)
    return [int(v) for v in d], [int(v) for v in n]


@pytest.mark.parametrize("name", list(CASES))
def test_parity_f32(name):
    H, N, B, T, U, R, L, p, ls, pct, wstd, tww, train = CASES[name]
    rng = np.random.default_rng(sum(name.encode()) + 1)
    tr = make_trainer(H, N, rounds=R, layers=L, dropout=p, labelsmooth=ls, pctteacherforcing=pct, window_std=wstd, train_with_window=tww)
    d, n = spread(rng, B, T, U)
    feat = torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32))
    for b in range(B):
        feat[b, :, :, d[b]:] = 0  # padded as the loader pads
    feat = feat.cuda()
    y, tsz = targets(rng, B, U, N, n)
    net_flat, crit_flat = tr.get_flat(0, 0).clone(), tr.get_flat(1, 0).clone()
    loss = tr.step(feat, torch.from_numpy(y).cuda(), train=train, input_sizes=d, target_sizes=tsz).cpu().numpy()
    torch.cuda.synchronize()
    enc = am_ref.RefNet(encoder_arch(H), F, N, net_flat, tr.layout(0), device="cpu")
    x = enc.forward(feat.cpu())
    tps, ups, bad = SR.frame_counts(d, x.shape[1], tsz, U)
    assert not any(bad) and min(tps) < 0.6 * x.shape[1] and max(tps) == x.shape[1]
    params = ref.unflatten(crit_flat, tr.layout(1), N, H, R, L)
    if train:
        seed = tr.seq2seq_seed()
        tokens = S.substituted_tokens(seed, y, N, pct)
        masks = [S.dropout_scales(seed, k, (B, U, H), p) for k in range(R * L)] if p > 0 else None
        want = SR.loss(params, x, y, N - 1, tokens, tps, ups, R, L, wstd if tww else 0.0, ls, masks)
    else:
        want = SR.loss(params, x, y, N - 1, ref.teacher_tokens(y, N), tps, ups, R, L, wstd, 0.0)
    assert max_rel(loss, want.detach().numpy()) < 1e-4, (loss, want)
    if not train:
        return
    want.sum().backward()
    got_c = tr.get_flat(1, 1).double().cpu()
    for i, (po, (off, k, _)) in enumerate(zip(params, tr.layout(1))):
        g = po.grad.reshape(-1).numpy()
        assert max_rel(got_c[off:off + k].numpy(), g) < 2e-4, (name, "criterion parameter", i, max_rel(got_c[off:off + k].numpy(), g))
    got_n = tr.get_flat(0, 1).double().cpu()
    for i, (po, (off, k, _)) in enumerate(zip(enc.params, tr.layout(0))):
        g = po.grad.reshape(-1).numpy()
        assert max_rel(got_n[off:off + k].numpy(), g) < 2e-4, (name, "encoder parameter", i, max_rel(got_n[off:off + k].numpy(), g))


def test_full_sizes_equal_no_sizes():
    """equal durations and every target size U: the step, the decode and the search give the unsized bits"""
    H, N, B, T, U = 32, 13, 3, 40, 8
    rng = np.random.default_rng(41)
    feat = torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32)).cuda()
    y, _ = targets(rng, B, U, N, [3, 7, 5])
    tgt = torch.from_numpy(y).cuda()
    a = make_trainer(H, N, maxlen=12, rounds=2, layers=2, window_std=3.0, train_with_window=True)
    b = make_trainer(H, N, maxlen=12, rounds=2, layers=2, window_std=3.0, train_with_window=True)
    b.set_flat(a.get_flat(0, 0), 0)
    b.set_flat(a.get_flat(1, 0), 1)
    la = a.step(feat, tgt)
    lb = b.step(feat, tgt, input_sizes=[T] * B, target_sizes=torch.full((B,), U, dtype=torch.int32, device="cuda"))
    assert torch.equal(la, lb)
    for w in (0, 1):
        assert torch.equal(a.get_flat(w, 1), b.get_flat(w, 1)) and torch.equal(a.get_flat(w, 0), b.get_flat(w, 0))
    for x, z in zip(a.decode(feat), b.decode(feat, input_sizes=[T] * B)):
        assert torch.equal(x, z)
    for K in (1, 4):
        for x, z in zip(a.beam_search(feat, K), b.beam_search(feat, K, input_sizes=[T] * B)):
            assert torch.equal(x, z)


# ---- on a given encoder output -------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def helper(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("s2s") / "criterion_sized.so")
    libdir = os.path.join(ROOT, "wav2letter_b200")
    import wav2letter_b200  # noqa: F401  (loads libw2l_b200.so)

    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "seq2seq_sizes", "criterion_sized.cpp"), "-o", so, "-L", libdir, "-l:libw2l_b200.so",
                    f"-Wl,-rpath,{libdir}"], check=True, capture_output=True)
    lib = ctypes.CDLL(so)
    lib.s2sCreate.restype = ctypes.c_void_p
    lib.s2sCreate.argtypes = [ctypes.c_int] * 6 + [ctypes.c_double, ctypes.c_int, ctypes.c_void_p]
    lib.s2sDestroy.argtypes = [ctypes.c_void_p]
    return lib


def P(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


class Crit:
    """Seq2SeqCriterion with seeded parameters (R rounds of L layers, eval or teacher forcing at 100 %, no dropout)"""

    def __init__(self, lib, H, N, maxlen, R=1, L=1, window_std=0.0, seed=0):
        g = torch.Generator().manual_seed(seed)
        shapes = ref.param_shapes(N, H, R, L)
        self.params = [(torch.rand(s, generator=g) * 2 - 1) / (H ** 0.5 if i not in (0, 1) else 1.0) for i, s in enumerate(shapes)]
        self.params[-2] *= 8.0  # sharper output distributions: decisions with clear margins
        self.dense = torch.cat([p.reshape(-1) for p in self.params]).cuda()
        self.lib, self.H, self.N, self.maxlen = lib, H, N, maxlen
        self.h = lib.s2sCreate(N, H, maxlen, R, L, 100, window_std, 1, P(self.dense))
        assert self.h

    def __del__(self):
        self.lib.s2sDestroy(ctypes.c_void_p(self.h))

    def forward(self, x, y, train, durations=None, tsz=None, grad=True):
        B, Tp, _ = x.shape
        loss = torch.empty(B, device="cuda")
        dx = torch.empty_like(x) if grad else None
        rc = self.lib.s2sForward(ctypes.c_void_p(self.h), int(train), P(x), B, Tp, P(y), y.shape[1], P(durations), P(tsz), P(loss), P(dx))
        assert rc == 0
        return loss, dx

    def decode(self, x, durations=None):
        B, Tp, _ = x.shape
        tok = torch.empty((B, self.maxlen), dtype=torch.int32, device="cuda")
        ln = torch.empty(B, dtype=torch.int32, device="cuda")
        assert self.lib.s2sDecode(ctypes.c_void_p(self.h), P(x), B, Tp, P(durations), P(tok), P(ln)) == 0
        vp = torch.empty_like(tok)
        assert self.lib.s2sViterbiPath(ctypes.c_void_p(self.h), P(x), B, Tp, P(durations), P(vp)) == 0
        assert torch.equal(vp, tok)
        return tok, ln

    def beam(self, x, K, durations=None):
        B, Tp, _ = x.shape
        out = (torch.empty((B, K, self.maxlen), dtype=torch.int32, device="cuda"), torch.empty((B, K), dtype=torch.int32, device="cuda"),
               torch.empty((B, K), device="cuda"), torch.empty(B, dtype=torch.int32, device="cuda"))
        assert self.lib.s2sBeam(ctypes.c_void_p(self.h), P(x), B, Tp, P(durations), K, self.maxlen, *[P(t) for t in out]) == 0
        return out


def padded_batch(rng, B, Tp, U, H, N, frames, tokens):
    x = torch.from_numpy(rng.standard_normal((B, Tp, 2 * H), dtype=np.float32)).cuda()
    y, tsz = targets(rng, B, U, N, tokens)
    d = torch.tensor([10 * f for f in frames], dtype=torch.int32, device="cuda")  # the longest spans T'
    return x, torch.from_numpy(y).cuda(), d, torch.tensor(tsz, dtype=torch.int32, device="cuda")


@pytest.mark.parametrize("mode", ["eval", "train", "eval_window", "train_window_r2s2"])
def test_truncation_bit_for_bit(helper, mode):
    """an utterance of a padded, sized batch: loss as its own frames and target alone, encoder gradient equal on its
    frames and exactly 0 beyond"""
    H, N, B, Tp, U = 32, 13, 4, 37, 11
    R, L = (2, 2) if "r2s2" in mode else (1, 1)
    c = Crit(helper, H, N, 12, R, L, 3.0 if "window" in mode else 0.0, seed=7)
    rng = np.random.default_rng(43)
    frames, tokens = [37, 20, 9, 1], [10, 4, 7, 2]
    x, y, d, tsz = padded_batch(rng, B, Tp, U, H, N, frames, tokens)
    train = mode.startswith("train")  # an eval forward has no gradient
    loss, dx = c.forward(x, y, train, d, tsz, grad=train)
    for b in range(B):
        xb, yb = x[b:b + 1, :frames[b]].contiguous(), y[b:b + 1, :tokens[b] + 1].contiguous()
        lb, dxb = c.forward(xb, yb, train, grad=train)
        assert torch.equal(loss[b:b + 1], lb), (mode, b, loss[b], lb)
        if not train:
            continue
        diff = (dx[b, :frames[b]] - dxb[0]).abs().max().item()
        assert torch.equal(dx[b, :frames[b]], dxb[0]), (mode, b, diff)
        assert (dx[b, frames[b]:] == 0).all()


def test_poisoned_padding_changes_nothing(helper):
    H, N, B, Tp, U = 32, 13, 4, 30, 9
    c = Crit(helper, H, N, 10, 2, 2, 3.0, seed=3)
    rng = np.random.default_rng(47)
    frames = [30, 17, 8, 2]
    x, y, d, tsz = padded_batch(rng, B, Tp, U, H, N, frames, [8, 3, 5, 1])
    xp = x.clone()
    for b, f in enumerate(frames):
        xp[b, f:] = float("nan")
    for train in (False, True):
        a, b_ = c.forward(x, y, train, d, tsz, grad=train), c.forward(xp, y, train, d, tsz, grad=train)
        assert torch.equal(a[0], b_[0]) and (not train or torch.equal(a[1], b_[1])), train
    for a, b_ in zip(c.decode(x, d), c.decode(xp, d)):
        assert torch.equal(a, b_)
    for K in (1, 4):
        for a, b_ in zip(c.beam(x, K, d), c.beam(xp, K, d)):
            assert torch.equal(a, b_)


@pytest.mark.parametrize("K", [1, 4, 16])
def test_decoding_is_each_utterance_alone(helper, K):
    """greedy decode and beam search of a mixed-length batch with sizes: the tokens, lengths and scores of a decode of
    each utterance's own frames, bit for bit"""
    H, N, B, Tp, maxlen = 32, 13, 5, 33, 10
    c = Crit(helper, H, N, maxlen, 2, 3, seed=11)
    rng = np.random.default_rng(53)
    frames = [33, 25, 12, 5, 1]
    x, _, d, _ = padded_batch(rng, B, Tp, 4, H, N, frames, [1] * B)
    bt, bl = c.decode(x, d)
    full = c.beam(x, K, d)
    for b, f in enumerate(frames):
        xb = x[b:b + 1, :f].contiguous()
        t1, l1 = c.decode(xb)
        assert torch.equal(bt[b:b + 1], t1) and torch.equal(bl[b:b + 1], l1), b
        for a, o in zip(full, c.beam(xb, K)):
            assert torch.equal(a[b:b + 1], o), (K, b)
    # and the float64 reference decodes the same tokens where its margins are clear
    params = [p.double() for p in c.params]
    xr = x.double().cpu()
    for b, (want, gaps) in enumerate(SR.greedy(params, xr, frames, N - 2, maxlen, 2, 3)):
        got = list(bt[b, :bl[b]].cpu().numpy())
        for i, (g_, w) in enumerate(zip(got, want)):
            if gaps[i] < 1e-3:
                break
            assert g_ == w, (b, i, got, want)


# ---- trainer ---------------------------------------------------------------------------------------------------
def test_trainer_decode_with_sizes_matches_the_criterion():
    """Trainer.decode with input_sizes decodes the trainer's encoder output as the float64 sized reference does, and
    Trainer.beam_search with K = 1 gives the same tokens"""
    H, N, B, T = 32, 13, 4, 40
    rng = np.random.default_rng(59)
    tr = make_trainer(H, N, maxlen=10, rounds=1, layers=2)
    crit = tr.get_flat(1, 0).clone()
    for i, (off, k, _) in enumerate(tr.layout(1)):  # seeded parameters with sharp output distributions and no eos
        v = torch.from_numpy(rng.uniform(-1, 1, k).astype(np.float32)) / (1.0 if i < 2 else H ** 0.5)
        crit[off:off + k] = v.cuda() * (8.0 if i == len(tr.layout(1)) - 2 else 1.0)
    crit[tr.layout(1)[-1][0] + N - 2] = -1e4
    tr.set_flat(crit, 1)
    feat = torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32)).cuda()
    d = [40, 31, 16, 3]
    tok, ln = tr.decode(feat, input_sizes=d)
    x = tr.forward(feat).double().cpu()
    params = ref.unflatten(tr.get_flat(1, 0), tr.layout(1), N, H, 1, 2)
    tps = SR.frame_counts(d, x.shape[1])[0]
    for b, (want, gaps) in enumerate(SR.greedy([p.detach() for p in params], x, tps, N - 2, 10, 1, 2)):
        got = list(tok[b, :ln[b]].cpu().numpy())
        for i, (g_, w) in enumerate(zip(got, want)):
            if gaps[i] < 1e-3:
                break
            assert g_ == w, (b, i, got, want)
    bt, bl, bs, bc = tr.beam_search(feat, 1, input_sizes=torch.tensor(d, dtype=torch.int32, device="cuda"))
    assert torch.equal(bt[:, 0], tok) and torch.equal(bl[:, 0], ln)


def test_bf16_with_loss_scaling():
    H, N, B, T, U = 32, 13, 4, 40, 9
    rng = np.random.default_rng(61)
    feat = torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32)).cuda()
    y, tsz = targets(rng, B, U, N, [8, 2, 5, 3])
    tgt = torch.from_numpy(y).cuda()
    d = [40, 22, 30, 9]
    a = make_trainer(H, N, precision="f32")
    b = make_trainer(H, N, precision="bf16", lr=0.01, lrcrit=0.01)
    b.set_flat(a.get_flat(0, 0), 0)
    b.set_flat(a.get_flat(1, 0), 1)
    la = a.step(feat, tgt, train=False, input_sizes=d, target_sizes=tsz).cpu().numpy()
    lb = b.step(feat, tgt, train=False, input_sizes=d, target_sizes=tsz).cpu().numpy()
    assert max_rel(lb, la) < 2e-2
    b.set_amp(True)
    for _ in range(3):
        assert torch.isfinite(b.step(feat, tgt, input_sizes=d, target_sizes=tsz)).all()
    assert b.skipped_steps() == 0


def test_rejection_and_refusals():
    from wav2letter_b200 import W2LError
    from wav2letter_b200.trainer import Trainer

    H, N, B, T, U = 32, 13, 3, 40, 8
    rng = np.random.default_rng(67)
    feat = torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32)).cuda()
    y, tsz = targets(rng, B, U, N, [5, 3, 6])
    tgt = torch.from_numpy(y).cuda()
    tr = make_trainer(H, N, lr=0.1, lrcrit=0.1)
    before = (tr.get_flat(0, 0).clone(), tr.get_flat(1, 0).clone())
    good = tr.step(feat, tgt, train=False, input_sizes=[40, 30, 20], target_sizes=tsz).cpu().numpy()
    cases = [([40, 0, 20], tsz), ([40, -5, 20], tsz), ([40, 30, 20], [tsz[0], 0, tsz[2]]), ([40, 30, 20], [tsz[0], U + 1, tsz[2]])]
    for d, t in cases:
        loss = tr.step(feat, tgt, input_sizes=d, target_sizes=t).cpu().numpy()
        assert np.isnan(loss[1]) and loss[0] == good[0] and loss[2] == good[2], (d, t, loss, good)
    loss = tr.step(feat, tgt, input_sizes=[0, 0, -1]).cpu().numpy()
    assert np.isnan(loss).all()
    assert tr.skipped_steps() == len(cases) + 1
    assert torch.equal(tr.get_flat(0, 0), before[0]) and torch.equal(tr.get_flat(1, 0), before[1])
    with pytest.raises(ValueError):
        tr.step(feat, tgt, input_sizes=[40, 30])
    for crit in ("ctc", "asg"):
        other = Trainer(encoder_arch(H), F, N, crit, lr=0.0)
        with pytest.raises(W2LError, match="seq2seq"):
            other.step(feat, torch.zeros((B, 4), dtype=torch.int32, device="cuda"), input_sizes=[40, 30, 20])


def test_launch_counts():
    """a sized step launches one size kernel more than an unsized one; a sized decode step launches what an unsized one does"""
    from wav2letter_b200 import capi

    H, N, B, T, U = 32, 13, 2, 40, 9
    rng = np.random.default_rng(71)
    tr = make_trainer(H, N, maxlen=16, rounds=2, layers=2)
    feat = torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32)).cuda()
    y, tsz = targets(rng, B, U, N, [8, 3])
    tgt = torch.from_numpy(y).cuda()
    isz = torch.tensor([40, 25], dtype=torch.int32, device="cuda")
    tsz = torch.tensor(tsz, dtype=torch.int32, device="cuda")

    def count(fn):
        fn()
        torch.cuda.synchronize()
        return {k: v[0] for k, v in capi.trace(fn).items()}

    plain = count(lambda: tr.step(feat, tgt))
    sized = count(lambda: tr.step(feat, tgt, input_sizes=isz, target_sizes=tsz))
    assert sized.pop("seq2seq_sizes_kernel") == 1
    assert sized == plain, (sized, plain)
    # every decode runs all 16 steps: eos can never win
    crit = tr.get_flat(1, 0).clone()
    crit[tr.layout(1)[-1][0] + N - 2] = -1e4
    tr.set_flat(crit, 1)
    plain = count(lambda: tr.decode(feat))
    sized = count(lambda: tr.decode(feat, input_sizes=isz))
    assert sized.pop("seq2seq_sizes_kernel") == 1
    assert sized == plain, (sized, plain)
