"""The streaming acoustic model (wav2letter_b200/streaming.py, w2l_stream_* in include/w2l_b200.h) on the BASELINE
streaming arch (recipes/streaming_convnets/librispeech/am_500ms_future_context.arch):

- the split of an utterance into chunks does not change a bit of its emissions (every output frame is the same per-row
  sum in the same order whatever the batch's row count);
- the concatenated emissions match the eval-mode whole-utterance forward of the training network and what the exported
  model gives under oracle/inference_ref.py (the in-tree inference library's arithmetic), within the export test's
  bound (the runtime always takes the one-warp-per-frame LayerNorm, the forward chooses by batch size);
- many streams with different start times, lengths and chunkings, interleaved in calls over varying subsets, each give
  their single-stream emissions bit for bit, also in batches of thousands of rows, and start makes a slot forget its
  past;
- the parameters are a snapshot taken at create; misuse is an error with text."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import inference_ref
from wav2letter_b200 import W2LError, archs
from wav2letter_b200.capi import _ptr, _stream, lib
from wav2letter_b200.streaming import StreamingAM
from wav2letter_b200.trainer import Trainer

pytestmark = pytest.mark.gpu

ARCH = archs.streaming_tds()


def make_trainer(N, precision, seed=0, steps=2, T=120):
    tr = Trainer(ARCH, 80, N, "ctc", "none", lr=0.05, precision=precision)
    g = torch.Generator(device="cuda").manual_seed(seed)
    feat = torch.randn((2, 1, 80, T), device="cuda", generator=g)
    tgt = torch.randint(0, N - 1, (2, 4), device="cuda", generator=g, dtype=torch.int32)
    for _ in range(steps):  # move the parameters (LayerNorm gains and biases included) off their initial values
        tr.step(feat, tgt, True)
    return tr


def features(T, seed, B=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn((B, 1, 80, T), device="cuda", generator=g)


def stream_utterance(am, x, chunk, slot=0):
    """x [1,1,80,T] fed in chunks of `chunk` frames, then finish; the concatenated emissions [T',N]"""
    T = x.shape[3]
    am.start([slot])
    parts = []
    for t0 in range(0, T, chunk):
        e, fo = am.run([slot], x[:, :, :, t0:t0 + chunk].contiguous())
        parts.append(e[0, :fo[0]].clone())
    e, fo = am.finish([slot])
    parts.append(e[0, :fo[0]].clone())
    return torch.cat(parts)


@pytest.mark.parametrize("precision", ["f32", "bf16"])
def test_chunking_does_not_change_a_bit(precision):
    N, T = 12, 211
    tr = make_trainer(N, precision)
    am = StreamingAM(tr, 1, max_chunk=T, precision=precision)
    x = features(T, 1)
    whole = stream_utterance(am, x, T)
    ref = tr.forward(x)[0]
    assert whole.shape == ref.shape
    for chunk in (1, 7, 50, 137):
        e = stream_utterance(am, x, chunk)
        assert torch.equal(e, whole), (chunk, float((e - whole).abs().max()))
    am.close()
    tr.close()


def test_equals_the_offline_network_and_the_inference_math(tmp_path):
    N, T = 12, 157
    tr = make_trainer(N, "f32", seed=4)
    am = StreamingAM(tr, 2, max_chunk=50, precision="f32")
    for seed in (5, 6):
        x = features(T, seed)
        e = stream_utterance(am, x, 50)
        ref = tr.forward(x)[0]
        assert e.shape == ref.shape
        bound = 2e-4 * float(ref.abs().max())
        diff = float((e - ref).abs().max())
        print(f"streaming vs offline forward (f32): max |diff| {diff:.3g}, bit-identical: {torch.equal(e, ref)}")
        assert diff <= bound, (diff, bound)
    out = str(tmp_path / "export")
    tr.export_streaming(out)
    x = features(T, 7)
    e = stream_utterance(am, x, 37).cpu().numpy()
    ref = inference_ref.run_export(out, x[0, 0].t().cpu().numpy())
    assert ref.shape == e.shape
    # the export test's bound (its absolute 1e-2, the converter's criterion, assumes unit-scale emissions; these reach
    # hundreds after the training steps, so the scale-relative bound is the one that applies)
    assert np.abs(ref - e).max() <= 2e-4 * max(1.0, np.abs(ref).max())
    am.close()
    tr.close()


def test_many_interleaved_streams_equal_their_single_stream_runs():
    N, S = 12, 64
    tr = make_trainer(N, "f32", seed=8)
    rng = np.random.default_rng(0)
    lens = [int(x) for x in rng.integers(1, 260, S)]
    chunks = [int(x) for x in rng.choice([1, 3, 7, 20, 50], S)]
    xs = [features(lens[s], 100 + s) for s in range(S)]
    single = StreamingAM(tr, 1, max_chunk=max(lens), precision="f32")
    refs = [stream_utterance(single, xs[s], lens[s]) for s in range(S)]
    am = StreamingAM(tr, S, max_chunk=50, precision="f32")
    # slot s starts at call begin[s]; a call serves a random subset of the live slots, each with its next chunk
    begin = [int(x) for x in rng.integers(0, 40, S)]
    pos = [0] * S
    outs = [[] for _ in range(S)]
    state = ["idle"] * S
    # slot 5 first runs an unrelated utterance part way; restarting it must forget that
    am.start([5])
    am.run([5], features(30, 999))
    call = 0
    while any(st != "done" for st in state):
        starting = [s for s in range(S) if state[s] == "idle" and begin[s] <= call]
        if starting:
            am.start(starting)
            for s in starting:
                state[s] = "live"
        live = [s for s in range(S) if state[s] == "live"]
        subset = [s for s in live if rng.random() < 0.7]
        if subset:
            fin = bool(rng.random() < 0.5)
            runs = [s for s in subset if pos[s] < lens[s]]
            if runs:
                Tc = max(min(chunks[s], lens[s] - pos[s]) for s in runs)
                x = torch.zeros((len(runs), 1, 80, Tc), device="cuda")
                frames = []
                for k, s in enumerate(runs):
                    n = min(chunks[s], lens[s] - pos[s])
                    x[k, :, :, :n] = xs[s][0, :, :, pos[s]:pos[s] + n]
                    frames.append(n)
                    pos[s] += n
                e, fo = am.run(runs, x, frames)
                for k, s in enumerate(runs):
                    outs[s].append(e[k, :fo[k]].clone())
            ends = [s for s in subset if pos[s] == lens[s]]
            if ends and fin:
                e, fo = am.finish(ends)
                for k, s in enumerate(ends):
                    outs[s].append(e[k, :fo[k]].clone())
                    state[s] = "done"
        call += 1
        assert call < 10000
    for s in range(S):
        got = torch.cat(outs[s])
        assert torch.equal(got, refs[s]), (s, got.shape, refs[s].shape)
    single.close()
    am.close()
    tr.close()


@pytest.mark.parametrize("precision", ["f32", "bf16"])
def test_large_batches_equal_single_stream_runs(precision):
    """96 streams of 37- and 50-frame chunks in every call: each layer's padded batch has thousands of rows, where
    w2l_layernorm_fwd would pick a different kernel than for one stream's few rows; the emissions must not change"""
    from wav2letter_b200 import streaming

    N, S = 12, 96
    tr = make_trainer(N, precision, seed=31)
    rng = np.random.default_rng(1)
    lens = [int(x) for x in rng.integers(120, 320, S)]
    chunks = [int(x) for x in rng.choice([37, 50], S)]
    _, first, _ = streaming.plan(ARCH, 80, N, [37])
    assert S * int(first[0, 0]) > 8 * 132  # past the row count where the automatic LayerNorm changes kernel on an H100
    xs = [features(lens[s], 300 + s) for s in range(S)]
    single = StreamingAM(tr, 1, max_chunk=max(lens), precision=precision)
    refs = [stream_utterance(single, xs[s], lens[s]) for s in range(S)]
    am = StreamingAM(tr, S, max_chunk=50, precision=precision)
    slots = list(range(S))
    am.start(slots)
    pos = [0] * S
    outs = [[] for _ in range(S)]
    while any(pos[s] < lens[s] for s in slots):
        x = torch.zeros((S, 1, 80, 50), device="cuda")
        frames = []
        for s in slots:
            n = min(chunks[s], lens[s] - pos[s])
            x[s, :, :, :n] = xs[s][0, :, :, pos[s]:pos[s] + n]
            frames.append(n)
            pos[s] += n
        e, fo = am.run(slots, x, frames)
        for s in slots:
            outs[s].append(e[s, :fo[s]].clone())
    e, fo = am.finish(slots)
    for s in slots:
        outs[s].append(e[s, :fo[s]].clone())
        got = torch.cat(outs[s])
        assert torch.equal(got, refs[s]), (s, got.shape, refs[s].shape)
    single.close()
    am.close()
    tr.close()


def test_parameters_are_a_snapshot():
    N, T = 12, 90
    tr = make_trainer(N, "f32", seed=11)
    am = StreamingAM(tr, 1, max_chunk=T, precision="f32")
    x = features(T, 12)
    before = stream_utterance(am, x, 30)
    am.start([0])
    e1, f1 = am.run([0], x[:, :, :, :45].contiguous())
    first = e1[0, :f1[0]].clone()
    tr.step(features(100, 13), torch.randint(0, N - 1, (1, 3), device="cuda", dtype=torch.int32), True)  # training goes on
    e2, f2 = am.run([0], x[:, :, :, 45:].contiguous())
    e3, f3 = am.finish([0])
    assert torch.equal(torch.cat([first, e2[0, :f2[0]], e3[0, :f3[0]]]), before)
    assert not torch.equal(tr.forward(x)[0], before)  # the trainer itself did move
    am.close()
    tr.close()


def test_full_size_head_chunked_equals_whole_and_offline():
    N, T = 10000, 300
    tr = make_trainer(N, "f32", seed=21, steps=1, T=100)
    am = StreamingAM(tr, 1, max_chunk=T, precision="f32")
    x = features(T, 22)
    whole = stream_utterance(am, x, T)
    assert torch.equal(stream_utterance(am, x, 50), whole)
    ref = tr.forward(x)[0]
    assert whole.shape == ref.shape
    assert float((whole - ref).abs().max()) <= 2e-4 * float(ref.abs().max())
    assert am.state_bytes > 0
    am.close()
    tr.close()


def test_misuse_is_an_error_with_text():
    N = 12
    bad = Trainer("V -1 NFEAT 1 0\nC2 1 4 5 1 2 1 -1 -1\nR\nLN 3\nV 0 320 1 0\nRO 1 0 3 2\nL 320 NLABEL\n", 80, N, "ctc")
    with pytest.raises(W2LError, match="unsupported LayerNorm axis"):
        StreamingAM(bad, 4)
    bad.close()
    tr = make_trainer(N, "tf32", steps=0)
    am = StreamingAM(tr, 4, max_chunk=100)
    x = features(100, 3)
    with pytest.raises(W2LError, match="out of range"):
        am.start([4])
    with pytest.raises(W2LError, match="not started"):
        am.run([1], x)
    am.start([0, 1])
    with pytest.raises(W2LError, match="listed twice"):
        am.run([0, 0], features(100, 3, B=2))
    with pytest.raises(W2LError, match="longer than Tc"):
        am.run([0], x, [101])
    with pytest.raises(W2LError, match="max_chunk"):
        am.run([0], features(101, 3))
    fo = (ctypes.c_int * 1)()
    small = torch.empty(8, device="cuda")
    rc = lib.w2l_stream_run(am.h, _stream(), 1, (ctypes.c_int * 1)(0), (ctypes.c_int * 1)(100), _ptr(x), 100, 0, _ptr(small), 8, fo)
    assert rc == 1 and b"capacity" in lib.w2l_last_error()
    am.finish([1], x)
    with pytest.raises(W2LError, match="finished"):
        am.run([1], x)
    am.start([1])
    am.run([1], x)  # started again: runs
    am.close()
    tr.close()
