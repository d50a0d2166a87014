"""The Seq2Seq criterion's beam search (Trainer.beam_search, Seq2SeqCriterion::beamSearch) on the GPU against the float64
search of tests/seq2seq_beam_reference.py.  Every parameter is drawn from seeded NumPy and set with set_flat, so the oracle's
decision margins are known before the GPU runs: each case asserts them >= 1e-3 first, then parity in f32 (counts,
order, tokens and lengths exactly, scores to 1e-4 of max(|score|, 1)), the termination paths, batch invariance,
K = 1 against the greedy decode, launch counts, the C++ call LPM makes, and the refusals."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import seq2seq_beam_reference as beamref
from oracle import am_ref
from oracle import seq2seq_ref as ref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = 16  # filterbanks of the test encoder: one strided C2 (T' = T / 2), then `L 2F 2H`
MARGIN = 1e-3


def encoder_arch(H):
    return f"V -1 NFEAT 1 0\nC2 1 2 5 1 2 1 -1 -1\nR\nV 0 {2 * F} 1 0\nRO 1 0 3 2\nL {2 * F} {2 * H}\n"


def draw(H, N, R, L, seed, eos_bias, wscale):
    """encoder and criterion parameters (float64 arrays in module / layout order) and the generator, which draws the features next"""
    rng = np.random.default_rng(seed)
    enc = [rng.uniform(-1, 1, n) / np.sqrt(fan) for n, fan in am_ref.param_shapes(encoder_arch(H), F, N)]
    crit = []
    for i, shp in enumerate(ref.param_shapes(N, H, R, L)):
        n = int(np.prod(shp))
        if i == 0:
            v = rng.uniform(-1, 1, n)  # E
        elif i == 1:
            v = rng.uniform(-0.5, 0.5, n)  # startEmbedding
        elif i == len(ref.param_shapes(N, H, R, L)) - 2:
            v = rng.uniform(-1, 1, n) * wscale / np.sqrt(H)  # W_o
        elif i == len(ref.param_shapes(N, H, R, L)) - 1:
            v = rng.uniform(-0.5, 0.5, n)  # b_o, with eos shifted so that completions come at different steps
            v[N - 2] += eos_bias
        else:
            v = rng.uniform(-1, 1, n) / np.sqrt(H)
        crit.append(v)
    return enc, crit, rng


def pack(arrays):
    """the trainer's arena: each parameter in a 16-byte aligned slot"""
    out = np.zeros(sum((a.size + 3) // 4 * 4 for a in arrays), np.float32)
    off = 0
    for a in arrays:
        out[off:off + a.size] = a.reshape(-1)
        off += (a.size + 3) // 4 * 4
    return out


def expected(H, N, B, T, R, L, K, maxlen, seed, eos_bias, wscale):
    """(enc, crit, features, per utterance (hyps, margins)) from the float64 encoder and search"""
    enc, crit, rng = draw(H, N, R, L, seed, eos_bias, wscale)
    feat = rng.standard_normal((B, 1, F, T), dtype=np.float32)
    net = am_ref.RefNet(encoder_arch(H), F, N, params=[torch.from_numpy(np.asarray(p, np.float32)) for p in enc], device="cpu")
    x = net.forward(torch.from_numpy(feat)).detach()
    params = [torch.from_numpy(np.asarray(p, np.float32).astype(np.float64)).reshape(s) for p, s in zip(crit, ref.param_shapes(N, H, R, L))]
    res = [beamref.beam(*beamref.model_step(params, x[b:b + 1], R, L), K, maxlen, N - 2) for b in range(B)]
    return enc, crit, feat, res


def make_trainer(H, N, maxlen, R=1, L=1, precision="f32"):
    from wav2letter_b200.trainer import Trainer

    cfg = dict(hidden=H, eos=N - 2, pad=N - 1, maxdecoderoutputlen=maxlen, rounds=R, layers=L)
    return Trainer(encoder_arch(H), F, N, "seq2seq", lr=0.0, precision=precision, seq2seq=cfg)


def gpu_trainer(H, N, R, L, maxlen, enc, crit, precision="f32"):
    tr = make_trainer(H, N, maxlen, R, L, precision)
    for which, arrays in ((0, enc), (1, crit)):
        flat = pack(arrays)
        assert flat.size == tr.num_params(which)
        tr.set_flat(torch.from_numpy(flat).cuda(), which)
    return tr


def check_parity(got, res, maxlen, pad):
    tokens, lengths, scores, counts = (t.cpu().numpy() for t in got)
    for b, (hyps, _margins) in enumerate(res):
        assert counts[b] == len(hyps), (b, counts[b], len(hyps))
        for k, (s, path) in enumerate(hyps):
            assert lengths[b, k] == len(path) and list(tokens[b, k, :len(path)]) == path, (b, k, tokens[b, k], path)
            assert (tokens[b, k, len(path):] == pad).all()
            assert abs(scores[b, k] - s) <= 1e-4 * max(abs(s), 1.0), (b, k, scores[b, k], s)
        assert (lengths[b, counts[b]:] == 0).all() and np.isneginf(scores[b, counts[b]:]).all()
        assert (tokens[b, counts[b]:] == pad).all()


# name: H, N, B, T, R, L, K, maxlen, seed, eos_bias, wscale (seeds whose oracle margins clear MARGIN)
CASES = {
    "small_k1_r1s1": (32, 13, 3, 40, 1, 1, 1, 10, 0, 1.0, 12.0),
    "small_k2_r1s1": (32, 13, 3, 40, 1, 1, 2, 10, 0, 1.0, 12.0),
    "small_k4_r1s1": (32, 13, 3, 40, 1, 1, 4, 10, 1, 1.0, 12.0),
    "small_k8_r1s1": (32, 13, 3, 40, 1, 1, 8, 10, 38, 1.0, 12.0),
    "small_k16_r1s1": (32, 13, 2, 40, 1, 1, 16, 4, 6, 1.0, 20.0),
    "small_k1_r2s3": (32, 13, 3, 40, 2, 3, 1, 10, 0, 1.0, 12.0),
    "small_k2_r2s3": (32, 13, 3, 40, 2, 3, 2, 10, 0, 1.0, 12.0),
    "small_k4_r2s3": (32, 13, 3, 40, 2, 3, 4, 10, 0, 1.0, 12.0),
    "small_k8_r2s3": (32, 13, 3, 40, 2, 3, 8, 10, 6, 1.0, 12.0),
    "small_k16_r2s3": (32, 13, 2, 40, 2, 3, 16, 4, 3, 1.0, 20.0),
}
CASES.update({
    # local_prior_match's proposal model: --encoderdim=512, 5000 word pieces + eos + pad, --lpmBeamsz=4, T' = 150
    "lpm": (512, 5002, 2, 300, 1, 1, 4, 150, 0, 8.0, 12.0),
    "n10002": (32, 10002, 2, 40, 1, 1, 4, 8, 0, 6.0, 12.0),
    "h1024": (1024, 13, 2, 40, 1, 1, 4, 20, 0, 3.0, 12.0),
})


@pytest.mark.parametrize("name", list(CASES))
def test_parity_f32(name):
    H, N, B, T, R, L, K, maxlen, seed, eb, ws = CASES[name]
    enc, crit, feat, res = expected(H, N, B, T, R, L, K, maxlen, seed, eb, ws)
    assert min(min(m) for _, m in res) >= MARGIN, [min(m) for _, m in res]
    tr = gpu_trainer(H, N, R, L, maxlen, enc, crit)
    check_parity(tr.beam_search(torch.from_numpy(feat).cuda(), K), res, maxlen, N - 1)


# name: eos_bias, seed, K, maxlen and what the oracle must show
TERMINATION = {
    "early_stop": (4.0, 5, 4, 40),
    "maxlen_no_completion": (-30.0, 0, 4, 8),
    "maxlen_some_completions": (0.0, 2, 4, 6),
}


@pytest.mark.parametrize("name", list(TERMINATION))
def test_termination(name):
    eb, seed, K, maxlen = TERMINATION[name]
    H, N, B, T = 32, 13, 2, 40
    enc, crit, feat, res = expected(H, N, B, T, 1, 1, K, maxlen, seed, eb, 6.0)
    assert min(min(m) for _, m in res) >= MARGIN
    for hyps, _ in res:
        lens = [len(p) for _, p in hyps]
        if name == "early_stop":  # K completions, all shorter than maxlen, sorted, and the search stopped on its own
            assert len(hyps) == K and max(lens) < maxlen - 1
            assert all(hyps[i][0] >= hyps[i + 1][0] for i in range(K - 1))
        elif name == "maxlen_no_completion":  # the live beam at length maxlen
            assert len(hyps) == K and lens == [maxlen] * K
        else:  # fewer than K completions, in completion order
            assert 0 < len(hyps) < K and max(lens) < maxlen
    if name == "maxlen_some_completions":
        assert any(len(h) > 1 for h, _ in res)
    tr = gpu_trainer(H, N, 1, 1, maxlen, enc, crit)
    check_parity(tr.beam_search(torch.from_numpy(feat).cuda(), K), res, maxlen, N - 1)


def test_batch_invariance():
    """a batch searches as each of its utterances alone, bit for bit"""
    H, N, B, T, K, maxlen = 32, 13, 5, 40, 4, 20
    enc, crit, rng = draw(H, N, 2, 3, 7, 1.0, 6.0)
    tr = gpu_trainer(H, N, 2, 3, maxlen, enc, crit)
    feat = torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32)).cuda()
    full = [t.cpu() for t in tr.beam_search(feat, K)]
    for b in range(B):
        one = [t.cpu() for t in tr.beam_search(feat[b:b + 1].contiguous(), K)]
        for a, o in zip(full, one):
            assert torch.equal(a[b:b + 1], o), b


@pytest.mark.parametrize("precision", ["f32", "bf16"])
def test_k1_is_greedy(precision):
    H, N, B, T, maxlen = 32, 13, 4, 40, 20
    enc, crit, rng = draw(H, N, 2, 3, 11, 1.0, 6.0)
    tr = gpu_trainer(H, N, 2, 3, maxlen, enc, crit, precision)
    feat = torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32)).cuda()
    gt, gl = tr.decode(feat)
    tokens, lengths, _scores, counts = tr.beam_search(feat, 1)
    assert (counts.cpu() == 1).all()
    assert torch.equal(lengths[:, 0].cpu(), gl.cpu()) and torch.equal(tokens[:, 0].cpu(), gt.cpu())


def test_kernel_counts_do_not_depend_on_length():
    from wav2letter_b200 import capi

    H, N, B, T, K = 32, 13, 2, 40, 4
    enc, crit, rng = draw(H, N, 2, 2, 13, -30.0, 6.0)  # no completion: every search runs to max_len
    tr = gpu_trainer(H, N, 2, 2, 100, enc, crit)
    feat = torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32)).cuda()
    per_step = {}
    for maxlen in (20, 100):
        tr.beam_search(feat, K, maxlen)  # warm
        torch.cuda.synchronize()
        got = capi.trace(lambda: tr.beam_search(feat, K, maxlen))
        counts = {k: v[0] for k, v in got.items() if "seq2seq" in k}
        assert counts["seq2seq_beam_init_kernel"] == 1 and counts["seq2seq_beam_finish_kernel"] == 1, counts
        per_step[maxlen] = {k: v / maxlen for k, v in counts.items() if k not in ("seq2seq_beam_init_kernel", "seq2seq_beam_finish_kernel")}
    assert per_step[20] == per_step[100], per_step
    assert per_step[20]["seq2seq_beam_topk_kernel"] == 1 and per_step[20]["seq2seq_gru_fwd_kernel"] == 4, per_step[20]


def test_cpp_beam_search_as_lpm_calls_it(tmp_path):
    """tests/seq2seq_beam/lpm_beam_search.cpp, compiled against fl_compat.h, runs local_prior_match's batchBeamSearch
    loop (one beamSearch per utterance from {CandidateHypo{}}, eos appended): the paths of Trainer.beam_search"""
    from wav2letter_b200 import capi

    H, N, B, T, K, maxlen = 32, 13, 3, 40, 4, 20
    enc, crit, rng = draw(H, N, 1, 1, 17, 1.0, 6.0)
    tr = gpu_trainer(H, N, 1, 1, maxlen, enc, crit)
    feat = torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32)).cuda()
    tokens, lengths, _scores, counts = (t.cpu().numpy() for t in tr.beam_search(feat, K))
    x = tr.forward(feat).contiguous()
    dense = torch.from_numpy(np.concatenate([np.asarray(p, np.float32).reshape(-1) for p in crit])).cuda()
    so = str(tmp_path / "lpm_beam_search.so")
    libdir = os.path.join(ROOT, "wav2letter_b200")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "seq2seq_beam", "lpm_beam_search.cpp"), "-o", so, "-L", libdir, "-l:libw2l_b200.so",
                    f"-Wl,-rpath,{libdir}"], check=True, capture_output=True)
    lib = ctypes.CDLL(so)
    cap = B * K * (maxlen + 1)
    paths = np.zeros(cap, np.int32)
    plen = np.zeros(B * K, np.int32)
    nums = np.zeros(B, np.int32)
    torch.cuda.synchronize()
    rc = lib.lpmBatchBeamSearch(ctypes.c_void_p(x.data_ptr()), B, x.shape[1], H, N, maxlen, ctypes.c_void_p(dense.data_ptr()),
                                capi.PRECISIONS["f32"], K, paths.ctypes.data_as(ctypes.c_void_p), plen.ctypes.data_as(ctypes.c_void_p),
                                nums.ctypes.data_as(ctypes.c_void_p))
    assert rc == 0
    i = 0
    for b in range(B):
        assert nums[b] == counts[b]
        for k in range(counts[b]):
            want = list(tokens[b, k, :lengths[b, k]]) + [N - 2]
            assert list(paths[i * (maxlen + 1): i * (maxlen + 1) + plen[i]]) == want, (b, k)
            i += 1


def test_errors():
    from wav2letter_b200 import W2LError, capi
    from wav2letter_b200.trainer import Trainer

    H, N, B, T = 32, 13, 2, 40
    rng = np.random.default_rng(19)
    feat = torch.from_numpy(rng.standard_normal((B, 1, F, T), dtype=np.float32)).cuda()
    tr = make_trainer(H, N, 10)
    for K in (0, 17):
        with pytest.raises(W2LError, match="beam size"):
            tr.beam_search(feat, K)
    ctc = Trainer(encoder_arch(H), F, N, "ctc", lr=0.0)
    with pytest.raises(W2LError, match="seq2seq"):
        ctc.beam_search(feat, 4, 10)
    K, L = 4, 10
    tokens = torch.empty((B, K, L), dtype=torch.int32, device="cuda")
    small = torch.empty(B, dtype=torch.int32, device="cuda")
    scores = torch.empty((B, K), dtype=torch.float32, device="cuda")
    rc = capi.lib.w2l_trainer_beam_search(tr.h, capi._stream(), B, T, capi._ptr(feat), K, L, capi._ptr(tokens), capi._ptr(small),
                                          capi._ptr(scores), capi._ptr(small), tokens.numel() - 1)
    assert rc == 1 and b"too small" in capi.lib.w2l_last_error()
    assert capi.lib.w2l_seq2seq_beam_init(None, B, 17, H, L, None, None, None, 0) == 4
