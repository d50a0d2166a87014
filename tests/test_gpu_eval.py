"""Scoring on the GPU (csrc/text_eval.cu, DESIGN.md §10): w2l_text_edit_counts against the host pipeline
(prediction2ltr / target2ltr / ltr2wrd / EditDistanceMeter) in all eight counts of every utterance, and
Trainer.evaluate against step(train=False), viterbi_path / decode and host scoring."""
import random
import zlib

import numpy as np
import pytest
import torch

import eval_reference as ref
from test_eval_cpu import GRID, host_counts, make

pytestmark = pytest.mark.gpu


def _dev(rows, fill):
    n = max([len(r) for r in rows] + [1])
    a = np.full((len(rows), n), fill, np.int32)
    for b, r in enumerate(rows):
        a[b, :len(r)] = r
    return torch.from_numpy(a).cuda()


def _check(tp, paths, targets, lengths=None):
    """device counts of padded rows against host scoring of each row"""
    pad = tp.pad_index
    P, Tg = _dev(paths, pad if tp.criterion == "seq2seq" else -1), _dev(targets, pad)
    Ln = None if lengths is None else torch.tensor(lengths, dtype=torch.int32, device="cuda")
    got = tp.edit_counts(P, Tg, Ln).cpu().numpy()
    for b in range(len(paths)):
        row = P[b].cpu().numpy() if lengths is None else paths[b][:lengths[b]]
        want = host_counts(tp, row, Tg[b].cpu().numpy())
        assert got[b].tolist() == want, (b, paths[b], targets[b])
    return got


@pytest.mark.parametrize("criterion,replabel,surround,wordpiece", GRID)
def test_counts_equal_host_scoring(criterion, replabel, surround, wordpiece):
    args = ref.pipeline_args(criterion, replabel, surround, wordpiece)
    tp, t = make(args), ref.Tables(**args)
    rng = random.Random(zlib.crc32(repr(("gpu", criterion, replabel, surround, wordpiece)).encode()))
    B = 200
    paths = [ref.random_row(rng, t, rng.randrange(0, 60), True) for _ in range(B)]
    targets = [ref.random_row(rng, t, rng.randrange(1, 30), False, invalid_rate=0.002, minus_one=0.005) for _ in range(B)]
    got = _check(tp, paths, targets)
    assert (got[:, 0] >= 0).sum() > B // 2
    # the same rows cut by path_lengths (host: the row's first lengths[b] entries)
    lengths = [rng.randrange(0, len(p) + 1) for p in paths]
    _check(tp, paths, targets, lengths)


def test_edge_cases():
    tp = make(ref.pipeline_args("ctc", 2, "|", False))
    t = ref.Tables(**ref.pipeline_args("ctc", 2, "|", False))
    ix = {e: i for i, e in enumerate(ref.LETTER_TOKENS)}
    a, b, c, sep = ix["a"], ix["b"], ix["c"], ix["|"]
    r1, r2 = t.role.index(1), t.role.index(2)
    cases = [
        ([], [a, b]),                            # empty hypothesis
        ([a, b], [sep]),                         # empty reference (the separator is trimmed away)
        ([], [sep]),                             # both empty
        ([t.blank] * 50, [a, sep, b]),           # all blank
        ([r1, a, b], [a, b]),                    # leading replabel: dropped
        ([a, r1, r2, b], [a, a, b]),             # doubled replabel: the second is dropped
        ([sep, a, sep, b, sep], [sep, a, b, sep]),  # <SIL> / surround at the ends
        ([a, -1, a, t.blank, -1, b], [a, a, b]),  # -1 inside a path
        ([a, b], [b, a]),                        # only the tie order decides the split: two substitutions
        ([a, t.N, b], [a, b]),                   # a token outside the dictionary: -1 counts
        ([a, b], [a, -1, b]),                    # -1 inside a target reaches the letters: the host throws
        ([a, b], [a, -2, -1, -1]),               # trailing negatives are padding
    ]
    got = _check(tp, [p for p, _ in cases], [q for _, q in cases])
    assert got[8].tolist()[:4] == [2, 0, 0, 2]
    assert (got[9] == -1).all() and (got[10] == -1).all() and got[11][0] == 1
    # seq2seq: rows without eos, eos in the middle, pad inside
    tp = make(ref.pipeline_args("seq2seq", 0, "", False))
    t = ref.Tables(**ref.pipeline_args("seq2seq", 0, "", False))
    _check(tp, [[a, b, c], [a, t.eos, b], [a, t.pad, b, t.eos, t.N], [t.eos]], [[a, b, t.eos], [a, t.eos], [c, t.pad, t.eos], [t.eos, t.pad]])


@pytest.mark.parametrize("B", [1, 7, 2000])
def test_batch_sizes_and_two_runs_same_bits(B):
    args = ref.pipeline_args("asg", 2, "|", True)
    tp, t = make(args), ref.Tables(**args)
    rng = random.Random(B)
    paths = [ref.random_row(rng, t, rng.randrange(0, 80), True) for _ in range(B)]
    targets = [ref.random_row(rng, t, rng.randrange(1, 30), False, invalid_rate=0.0) for _ in range(B)]
    got = _check(tp, paths, targets)
    P, Tg = _dev(paths, -1), _dev(targets, -1)
    assert np.array_equal(tp.edit_counts(P, Tg).cpu().numpy(), got)


@pytest.mark.parametrize("ref_len", [20, 600, 12000])
def test_long_hypotheses(ref_len):
    """10 500 letters against short and long references; against itself (90 % kept) it runs past the on-chip diagonals"""
    args = ref.pipeline_args("ctc", 0, "", False)
    tp, t = make(args), ref.Tables(**args)
    rng = random.Random(ref_len)
    letters = [ref.LETTER_TOKENS.index(x) for x in "abcé中|"]
    hyp = [rng.choice(letters) for _ in range(10500)]
    path = [v for x in hyp for v in (x, t.blank)]
    tgt = [rng.choice(letters) for _ in range(ref_len)]
    if ref_len > 10000:
        tgt = [x if rng.random() < 0.9 else rng.choice(letters) for x in hyp[:ref_len]]
    _check(tp, [path, path[:100]], [tgt, tgt])


def test_limit_is_refused_before_launch():
    from wav2letter_b200 import W2LError
    from wav2letter_b200.capi import lib

    tp = make(ref.pipeline_args("ctc", 0, "", False))  # one letter per token, no replabel: the limit is the width
    lim = 1 << 20
    P = torch.full((1, lim), tp.num_classes - 1, dtype=torch.int32, device="cuda")
    Tg = torch.full((1, 4), ref.LETTER_TOKENS.index("a"), dtype=torch.int32, device="cuda")
    assert tp.edit_counts(P, Tg).cpu().tolist() == [[4, 4, 0, 0, 1, 1, 0, 0]]
    P = torch.full((1, lim + 1), tp.num_classes - 1, dtype=torch.int32, device="cuda")
    counts_before = lib.w2l_launch_count()
    with pytest.raises(W2LError) as e:
        tp.edit_counts(P, Tg)
    assert e.value.code == 4 and lib.w2l_launch_count() == counts_before
    tp2 = make(ref.pipeline_args("ctc", 2, "", True))  # 3 x (1 + 2) letters per entry
    with pytest.raises(W2LError):
        tp2.edit_counts(torch.zeros((1, lim // 9 + 1), dtype=torch.int32, device="cuda"), Tg)


# ---- Trainer.evaluate --------------------------------------------------------------------------------------------------
def _host_rows(tp, paths, targets):
    return np.array([host_counts(tp, p, q) for p, q in zip(paths.cpu().numpy(), targets.cpu().numpy())], np.int32)


def _ctc_asg_trainer(criterion, arch, N):
    import test_gpu_slimipl as sl

    return sl._trainer(criterion, N=N, lr=0.05, momentum=0.9, maxgradnorm=1.0, arch=arch)


@pytest.mark.parametrize("criterion", ["ctc", "asg"])
def test_evaluate_ctc_asg(criterion):
    import test_gpu_convglu as cg
    import test_gpu_slimipl as sl
    from wav2letter_b200.text import ErrorRates, TextPipeline

    # TDS + CTC, and conv_glu + ASG with the recipes' --replabel=2 --surround=|
    text = TextPipeline(sl.LETTERS, "", criterion, 0 if criterion == "ctc" else 2, "" if criterion == "ctc" else "|", False, "|")
    tr = _ctc_asg_trainer(criterion, sl.TDS_ARCH if criterion == "ctc" else cg.ARCH, text.num_classes)
    rng = np.random.default_rng(3)
    feat = sl._spoken(rng, text, sl.TRANSCRIPTS)
    tgt = torch.from_numpy(text.encode_batch(sl.TRANSCRIPTS)).cuda()
    for i in range(60):
        loss, counts = tr.evaluate(feat, tgt, text)
        assert torch.equal(loss, tr.step(feat, tgt, train=False))
        assert np.array_equal(counts.cpu().numpy(), _host_rows(text, tr.viterbi_path(feat), tgt))
        if (counts[:, 1:4].sum() + counts[:, 5:8].sum()).item() == 0:
            break
        for _ in range(50):
            tr.step(feat, tgt, total_batch=3.0)
    # overfitted: its own transcripts score no errors
    assert counts[:, 1:4].sum().item() == 0 and counts[:, 5:8].sum().item() == 0
    m = ErrorRates()
    m.add(counts)
    assert m.ter() == 0.0 and m.wer() == 0.0 and m.value()[1][1] == sum(len(s.split()) for s in sl.TRANSCRIPTS)
    tr.close()


def test_evaluate_seq2seq_padded_batch():
    import test_gpu_seq2seq as s2s
    from wav2letter_b200.text import ErrorRates, TextPipeline

    tokens = "|\n" + "\n".join("abcdefg") + "\n"
    text = TextPipeline(tokens, "", "seq2seq", 0, "", False, "|")
    N = text.num_classes
    tr = s2s.make_trainer(32, N, maxlen=12, lr=0.05, lrcrit=0.05)
    rng = np.random.default_rng(5)
    B, T = 4, 40
    feat = s2s.features(rng, B, T)
    tgt = torch.from_numpy(s2s.targets(rng, B, 8, N)).cuda()
    isz, tsz = [40, 31, 22, 40], [int((r != N - 1).sum()) for r in tgt.cpu().numpy()]
    for _ in range(3):
        tr.step(feat, tgt, input_sizes=isz, target_sizes=tsz)
    loss, counts = tr.evaluate(feat, tgt, text, input_sizes=isz, target_sizes=tsz)
    assert torch.equal(loss, tr.step(feat, tgt, train=False, input_sizes=isz, target_sizes=tsz))
    tokens_, _ = tr.decode(feat, input_sizes=isz)
    assert np.array_equal(counts.cpu().numpy(), _host_rows(text, tokens_, tgt))
    # unsized, and decode rows cut by their lengths give the same counts as whole rows
    loss, counts = tr.evaluate(feat, tgt, text)
    assert torch.equal(loss, tr.step(feat, tgt, train=False))
    tokens_, lengths = tr.decode(feat)
    assert np.array_equal(counts.cpu().numpy(), _host_rows(text, tokens_, tgt))
    assert torch.equal(text.edit_counts(tokens_, tgt, lengths), counts)
    m = ErrorRates()
    m.add(counts)
    m.add(torch.full((1, 8), -1, dtype=torch.int32, device="cuda"))
    assert m.value()[2] == 1 and m.value()[0][1] == int(counts[:, 0].sum())
    # a ctc trainer takes no sizes
    from wav2letter_b200 import W2LError

    ctc_text = TextPipeline(tokens, "", "ctc", 0, "", False, "|")
    ctc = _ctc_asg_trainer("ctc", __import__("test_gpu_slimipl").TDS_ARCH, ctc_text.num_classes)
    with pytest.raises(W2LError):
        ctc.evaluate(s2s.features(rng, 2, 40), torch.zeros((2, 3), dtype=torch.int32, device="cuda"), ctc_text, input_sizes=[40, 30])
    tr.close()
    ctc.close()


# ---- fl_compat: DeviceEditScorer -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def scorer_lib(tmp_path_factory):
    import ctypes
    import os
    import subprocess

    import wav2letter_b200  # noqa: F401  (loads libw2l_b200.so)

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    so = str(tmp_path_factory.mktemp("scorer") / "scorer.so")
    libdir = os.path.join(root, "wav2letter_b200")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-I", os.path.join(root, "include"),
                    os.path.join(root, "tests", "text_eval", "scorer.cpp"), "-o", so, "-L", libdir, "-l:libw2l_b200.so",
                    f"-Wl,-rpath,{libdir}"], check=True, capture_output=True)
    lib = ctypes.CDLL(so)
    vp, i, cp = ctypes.c_void_p, ctypes.c_int, ctypes.c_char_p
    lib.scorerCreate.restype = vp
    lib.scorerCreate.argtypes = [cp, cp, i, cp, i, cp]
    lib.scorerDestroy.argtypes = [vp]
    lib.scorerCompare.argtypes = [vp, vp, vp, i, i, vp, vp, i, vp]
    return lib


@pytest.mark.parametrize("criterion,replabel,surround,wordpiece", [("ctc", 0, "", True), ("asg", 2, "|", False), ("seq2seq", 0, "", False)])
def test_fl_compat_scorer_equals_the_per_utterance_loop(scorer_lib, criterion, replabel, surround, wordpiece):
    import ctypes

    args = ref.pipeline_args(criterion, replabel, surround, wordpiece)
    t = ref.Tables(**args)
    h = scorer_lib.scorerCreate(("\n".join(args["tokens"]) + "\n").encode(), criterion.encode(), replabel, surround.encode(), int(wordpiece),
                                args["wordsep"].encode())
    assert h
    rng = random.Random(zlib.crc32(repr(("fl", criterion)).encode()))
    pad = t.pad if criterion == "seq2seq" else -1
    for k in range(6):
        B = rng.choice([1, 5, 64])
        paths = [ref.random_row(rng, t, rng.randrange(0, 50), True, invalid_rate=0.0) for _ in range(B)]
        targets = [ref.random_row(rng, t, rng.randrange(1, 20), False, invalid_rate=0.0, minus_one=0.0) for _ in range(B)]
        if k == 5:
            paths[B // 2] = [0, t.N, 1]  # a token outside the dictionary: both refuse the batch
        P, Tg = _dev(paths, pad), _dev(targets, pad)
        Ph, Th = P.cpu().numpy(), Tg.cpu().numpy()
        out = (ctypes.c_longlong * 20)()
        rc = scorer_lib.scorerCompare(ctypes.c_void_p(h), ctypes.c_void_p(P.data_ptr()), Ph.ctypes.data_as(ctypes.c_void_p), B, P.shape[1],
                                      ctypes.c_void_p(Tg.data_ptr()), Th.ctypes.data_as(ctypes.c_void_p), Tg.shape[1], out)
        v = list(out)
        if k == 5:
            assert rc == 3 and v[:10] == [0] * 10
        else:
            assert rc == 0 and v[:10] == v[10:] and v[1] > 0
    scorer_lib.scorerDestroy(ctypes.c_void_p(h))
