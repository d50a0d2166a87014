"""The streaming MFSC front end (wav2letter_b200.streaming.StreamingFeatures, w2l_mfsc_stream_* in include/w2l_b200.h):

- the split of a stream into chunks does not change a bit of its features, and every call's frame count is
  LogMelFeature::run's buffer arithmetic;
- each of 64 or 1024 streams with random chunks and staggered starts gives its single-stream features bit for bit, also
  at the frame lengths where w2l_gemm would split K (48 kHz x 25 ms, 16 kHz x 64 ms) if the DFT let it;
- a whole stream equals w2l_mfsc(..., left_ctx) of the utterance up to the order of the double window sums;
- the precision setting is ignored, start forgets, misuse is an error with text;
- audio -> StreamingFeatures -> StreamingAM gives emissions that do not depend on the chunking or the other streams, and
  match the whole-utterance Trainer.forward of w2l_mfsc's features."""
import ctypes

import numpy as np
import pytest
import torch

import features_reference as R
from test_gpu_features import synth
from test_gpu_streaming import make_trainer
from wav2letter_b200 import W2LError, capi
from wav2letter_b200.capi import _ptr, _stream, lib
from wav2letter_b200.features import mfsc
from wav2letter_b200.streaming import StreamingAM, StreamingFeatures

pytestmark = pytest.mark.gpu


def ints(*v):
    return (ctypes.c_int * len(v))(*v)


def frames_of(avail, frame, stride):
    return 0 if avail < frame else 1 + (avail - frame) // stride


def audio_of(n, seed, fs=16000):
    x = synth(n, seed) if fs == 16000 else np.interp(np.arange(n) * 16000 / fs, np.arange(n), synth(n, seed))
    return torch.from_numpy(x.astype(np.float32)).cuda()


def feed(fe, x, sizes, slot=0, check_frames=True):
    """x [S] fed in calls of `sizes` samples (the last one finishing), alone in slot `slot`: the features [F, T]"""
    fe.start([slot])
    frame, stride = fe_geom(fe)
    held, parts, pos = 0, [], 0
    for k, c in enumerate(sizes):
        chunk = x[pos:pos + c][None].contiguous() if c > 0 else None
        f, fo = fe.run([slot], chunk, [c], finish=k == len(sizes) - 1)
        want = frames_of(held + c, frame, stride)
        if check_frames:
            assert fo == [want], (k, c, fo, want)
        held += c - want * stride
        pos += c
        parts.append(f[0, 0, :, :fo[0]].clone())
    assert pos == len(x)
    return torch.cat(parts, 1)


def fe_geom(fe):
    return R.frame_samples(fe.sample_rate, fe.frame_ms), R.frame_samples(fe.sample_rate, fe.stride_ms)


def make(max_streams, max_chunk, fs=16000, frame_ms=25, stride_ms=10, n_filters=80, left_ctx=300):
    return StreamingFeatures(max_streams, max_chunk, n_filters, left_ctx, fs, frame_ms, stride_ms)


def test_chunking_does_not_change_a_bit():
    fe = make(1, 65535)
    frame, stride = fe_geom(fe)
    n = 3 * 16000 + 77
    x = audio_of(n, 1)
    whole = feed(fe, x, [n])
    assert whole.shape == (80, frames_of(n, frame, stride))
    rest = n - (1 + frame - 1 + frame + 8000)
    a = [0, 1, frame - 1, frame, 8000, 0] + [8000] * (rest // 8000) + [rest % 8000]
    b = [160] * (n // 160) + [n % 160]
    rng = np.random.default_rng(0)
    c = []
    while sum(c) < n:
        c.append(int(min(rng.integers(0, 3000), n - sum(c))))
    for sizes in (a, b, c, [n, 0]):
        got = feed(fe, x, sizes)
        assert torch.equal(got, whole), sizes[:8]
    fe.close()


def run_interleaved(fe, xs, rng, max_chunk):
    """every stream starts at a random call and is fed random chunks in calls that serve all live streams"""
    S = len(xs)
    begin = [int(v) for v in rng.integers(0, 6, S)]
    pos, outs, live, done = [0] * S, [[] for _ in range(S)], [False] * S, [False] * S
    call = 0
    while not all(done):
        starting = [s for s in range(S) if not live[s] and not done[s] and begin[s] <= call]
        if starting:
            fe.start(starting)
            for s in starting:
                live[s] = True
        slots = [s for s in range(S) if live[s]]
        if slots:
            sizes = [int(min(rng.integers(0, max_chunk + 1), len(xs[s]) - pos[s])) for s in slots]
            Sc = max(sizes)
            audio = torch.zeros((len(slots), Sc), device="cuda")
            for i, s in enumerate(slots):
                audio[i, :sizes[i]] = xs[s][pos[s]:pos[s] + sizes[i]]
            last = [pos[s] + sizes[i] == len(xs[s]) for i, s in enumerate(slots)]
            # streams at their end finish in a call of their own, the others run together
            for group, fin in (([i for i in range(len(slots)) if not last[i]], False), ([i for i in range(len(slots)) if last[i]], True)):
                if not group:
                    continue
                a = audio[group].contiguous() if Sc > 0 else None
                f, fo = fe.run([slots[i] for i in group], a, [sizes[i] for i in group], finish=fin)
                for j, i in enumerate(group):
                    outs[slots[i]].append(f[j, 0, :, :fo[j]].clone())
            for i, s in enumerate(slots):
                pos[s] += sizes[i]
                if last[i]:
                    live[s], done[s] = False, True
        call += 1
    return [torch.cat(o, 1) for o in outs]


@pytest.mark.parametrize("S", [64, 1024])
@pytest.mark.parametrize("fs,frame_ms", [(16000, 25), (48000, 25), (16000, 64)])
def test_batching_does_not_change_a_bit(S, fs, frame_ms):
    if S == 1024 and (fs, frame_ms) == (16000, 64):
        pytest.skip("the two split-K shapes are covered at 1024 streams by 48 kHz")
    rng = np.random.default_rng(S + fs + frame_ms)
    max_chunk = 8000 if fs == 16000 else 24000
    lens = [int(v) for v in rng.integers(1, 4 * max_chunk, S)]
    xs = [audio_of(lens[s], 1000 + s, fs) for s in range(S)]
    single = make(1, 65535, fs, frame_ms)
    refs = [feed(single, xs[s], [60000] * (lens[s] // 60000) + [lens[s] % 60000]) for s in range(S)]
    fe = make(S, max_chunk, fs, frame_ms)
    outs = run_interleaved(fe, xs, rng, max_chunk)
    for s in range(S):
        assert torch.equal(outs[s], refs[s]), (s, lens[s])
    fe.close()
    single.close()


@pytest.mark.parametrize("left_ctx", [1, 7, 300])
def test_equals_the_offline_path(left_ctx):
    n = 5 * 16000 + 311
    x = audio_of(n, 20 + left_ctx)
    fe = make(2, 8000, left_ctx=left_ctx)
    got = feed(fe, x, [8000] * (n // 8000) + [n % 8000])
    off, (T,) = mfsc(x[None].contiguous(), [n], left_ctx=left_ctx)
    assert got.shape == (80, T)
    diff = float((got - off[0, 0]).abs().max())
    print(f"streaming vs w2l_mfsc, left_ctx {left_ctx}: max |diff| {diff:.3g}")
    assert diff <= 1e-6
    ref = R.mfsc_utterance(R.Params(16000, 25, 10, 80), x.double().cpu().numpy(), left_ctx)
    assert np.abs(got.cpu().numpy() - ref.T).max() <= 1e-4
    # silence: zeros; a window longer than the stream so far (the first call's frames) is what the offline path does
    z = feed(fe, torch.zeros(8000, device="cuda"), [8000], slot=1)
    assert z.shape[1] > 0 and (z == 0).all()
    fe.close()


def test_the_precision_setting_is_ignored():
    n = 40000
    x = audio_of(n, 3)
    sizes = [3000] * (n // 3000) + [n % 3000]
    prev = capi.get_precision()
    outs = []
    try:
        for p in ("tf32", "f32", "bf16"):
            capi.set_precision(p)
            fe = make(1, 8000)
            outs.append(feed(fe, x, sizes))
            fe.close()
    finally:
        capi.set_precision(prev)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


def test_start_forgets_and_misuse_is_an_error():
    fe = make(4, 8000)
    x = audio_of(30000, 4)
    fresh = feed(fe, x, [8000, 8000, 8000, 6000], slot=2)
    fe.start([3])
    fe.run([3], audio_of(7777, 5)[None].contiguous())  # slot 3 holds samples and sums of another stream
    assert torch.equal(feed(fe, x, [8000, 8000, 8000, 6000], slot=3), fresh)
    one = torch.zeros((1, 100), device="cuda")
    with pytest.raises(W2LError, match="finished"):
        fe.run([3], one)
    with pytest.raises(W2LError, match="not started"):
        fe.run([0], one)
    fe.start([0, 1])
    with pytest.raises(W2LError, match="out of range"):
        fe.run([4], one)
    with pytest.raises(W2LError, match="listed twice"):
        fe.run([0, 0], torch.zeros((2, 100), device="cuda"))
    with pytest.raises(W2LError, match="longer than Sc"):
        fe.run([0], one, [101])
    with pytest.raises(W2LError, match="Sc must be"):
        fe.run([0], torch.zeros((1, 8001), device="cuda"))
    # a feature buffer one frame short: 8000 new samples give 1 + (8000 - 400) // 160 = 48 frames
    big = torch.zeros((1, 8000), device="cuda")
    assert lib.w2l_mfsc_stream_run(fe.h, _stream(), 1, ints(1), ints(8000), _ptr(big), 8000, 0, _ptr(big), 80 * 47, (ctypes.c_int * 1)()) == 1
    assert b"capacity" in lib.w2l_last_error()
    assert fe.state_bytes == 4 * 2 * 400 + 16 * 2 * 300
    fe.close()


@pytest.mark.parametrize("precision", ["f32", "bf16"])
def test_audio_to_emissions_end_to_end(precision):
    N, ell = 12, 300
    tr = make_trainer(N, precision, seed=3)
    fe = make(8, 8000, left_ctx=ell)
    am = StreamingAM(tr, 8, max_chunk=fe.max_frames_out, precision=precision)
    lens = [41000, 17123, 30000]
    xs = [audio_of(n, 60 + k) for k, n in enumerate(lens)]

    def through(slots, chunks):
        """streams xs[k] in slots[k], fed together call by call (chunks[k]: sizes); the emissions per stream"""
        fe.start(slots)
        am.start(slots)
        pos = [0] * len(slots)
        outs = [[] for _ in slots]
        for c in range(max(len(ch) for ch in chunks)):
            sizes = [ch[c] if c < len(ch) else 0 for ch in chunks]
            fin = c == max(len(ch) for ch in chunks) - 1
            Sc = max(sizes)
            audio = torch.zeros((len(slots), Sc), device="cuda") if Sc else None
            for k in range(len(slots)):
                if sizes[k]:
                    audio[k, :sizes[k]] = xs[k][pos[k]:pos[k] + sizes[k]]
                pos[k] += sizes[k]
            feats, frames = fe.run(slots, audio, sizes, finish=fin)
            e, fo = am.run(slots, feats, frames, finish=fin)
            for k in range(len(slots)):
                outs[k].append(e[k, :fo[k]].clone())
        return [torch.cat(o) for o in outs]

    def split(n, c):
        return [c] * (n // c) + [n % c]

    # first call: 100 samples each, no stream completes a frame (features [n,1,F,0])
    one = through([0, 1, 2], [[100] + split(n - 100, 8000) for n in lens])
    two = through([5, 3, 7], [[0, 399, 1] + split(n - 400, 1777) for n in lens])
    alone = [through([4], [split(n, 5000)])[0] for n in lens[:1]]
    for k in range(3):
        assert torch.equal(one[k], two[k]), k
    assert torch.equal(one[0], alone[0])
    if precision == "f32":
        for k, n in enumerate(lens):
            feats, _ = mfsc(xs[k][None].contiguous(), [n], left_ctx=ell)
            ref = tr.forward(feats)[0]
            assert one[k].shape == ref.shape
            diff, bound = float((one[k] - ref).abs().max()), 2e-4 * float(ref.abs().max())
            print(f"audio -> emissions vs whole-utterance forward (f32): max |diff| {diff:.3g} (bound {bound:.3g})")
            assert diff <= bound
    am.close()
    fe.close()
    tr.close()
