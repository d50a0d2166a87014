"""The criterion's path of the streaming acoustic model (StreamingAM.run(..., path=True), w2l_stream_run_path) on the
BASELINE streaming arch:

- per stream, the committed entries of every call and of finish put end to end are, bit for bit, the criterion's
  viterbiPath of its streaming emissions put end to end: w2l_argmax_path for CTC, w2l_fcc_viterbi (N <= 32) /
  w2l_fcc_viterbi64 (N <= 64) for ASG and LinSeg; over 1-frame chunks, calls that give no output frame and a finish
  with no new data; without the emission copy too; path_info matches the host's count of the same entries;
- the path does not change with the chunking, the slot or the other streams of a call (up to 1024, staggered starts,
  a start that restarts a running slot);
- two states tied forever force commits, whose count and labels match the NumPy model
  (tests/streaming_path_reference.py);
- the joined path gives TextPipeline the words of the whole-utterance path;
- bad arguments are refused before anything is launched."""
import numpy as np
import pytest
import torch

from streaming_path_reference import CarriedViterbi, tied_forever
from wav2letter_b200 import W2LError, archs, capi
from wav2letter_b200.streaming import StreamingAM
from wav2letter_b200.text import TextPipeline
from wav2letter_b200.trainer import Trainer

pytestmark = pytest.mark.gpu

ARCH = archs.streaming_tds()
LETTERS = "|\n'\n" + "\n".join("abcdefghijklmnopqrstuvwxyz") + "\n"  # 28 tokens


def make_trainer(crit, N, seed=0, precision="f32"):
    tr = Trainer(ARCH, 80, N, crit, "none", precision=precision)
    if crit != "ctc":  # transitions off their zero start, so the recursion has something to carry
        g = torch.Generator(device="cuda").manual_seed(seed)
        tr.set_flat(torch.randn((N * N,), device="cuda", generator=g), which=1)
    return tr


def transitions(tr):
    N = tr.n_label
    return tr.get_flat(1)[: N * N].view(N, N).contiguous()


def features(T, seed, B=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn((B, 1, 80, T), device="cuda", generator=g)


def viterbi(tr, emis):
    """the criterion's whole-utterance viterbiPath of emis [T, N]"""
    if tr.criterion == "ctc":
        return capi.argmax_path(emis[None].contiguous())[0]
    fn = capi.fcc_viterbi if tr.n_label <= 32 else capi.fcc_viterbi64
    return fn(emis[None].contiguous(), transitions(tr))[0]


def stream_path(am, x, chunks, slot=0, emissions=True):
    """x [1,1,80,T] in calls of `chunks` frames (0 allowed), then finish with no new data.  Returns (joined emissions or
    None, joined path, per call (frames_out, path_info))."""
    am.start([slot])
    es, ps, infos, t0 = [], [], [], 0
    for c in list(chunks) + [None]:
        if c is None:
            e, fo, p, info = am.finish([slot], path=True, emissions=emissions)
        else:
            xc = x[:, :, :, t0:t0 + c].contiguous()
            t0 += c
            e, fo, p, info = am.run([slot], xc if c else None, path=True, emissions=emissions)
        info = info.cpu()
        if emissions:
            es.append(e[0, :fo[0]].clone())
        ps.append(p[0, :int(info[0, 1])].clone())
        infos.append((fo[0], info[0].tolist()))
    assert t0 == x.shape[3]
    return (torch.cat(es) if emissions else None), torch.cat(ps), infos


def check_info(tr, infos, n_frames):
    """path_info against the host's count: frame indices follow each other, every frame is committed once, nothing is
    forced; CTC commits every output frame in its own call"""
    done = 0
    for fo, (first, count, forced) in infos:
        assert first == done and forced == 0
        if tr.criterion == "ctc":
            assert count == fo
        done += count
    assert done == n_frames


CASES = [("ctc", 30), ("ctc", 10000), ("asg", 2), ("asg", 30), ("asg", 32), ("asg", 33), ("asg", 64), ("linseg", 30), ("linseg", 64)]


@pytest.mark.parametrize("crit,N", CASES)
def test_joined_path_is_the_viterbi_path(crit, N):
    T = 173
    tr = make_trainer(crit, N, seed=N)
    am = StreamingAM(tr, 2, max_chunk=T, precision="f32")
    assert am.max_path_out == (am.max_frames_out if crit == "ctc" else 1024 + am.max_frames_out)
    x = features(T, N)
    rng = np.random.default_rng(N)
    ref_path = None
    rand = [int(c) for c in np.minimum(rng.integers(0, 12, 20), T)]
    while sum(rand) > T:
        rand.pop()
    for chunks in ([T], [1] * T, [0, 3, 0, 5, 1, 1, 40, 0, 2, 121], rand + [T - sum(rand)]):
        e, p, infos = stream_path(am, x, chunks)
        want = viterbi(tr, e)
        assert torch.equal(p, want), chunks
        check_info(tr, infos, e.shape[0])
        if ref_path is None:
            ref_path = p
        assert torch.equal(p, ref_path), chunks  # the same bits whatever the chunking
        if 1 in chunks:
            assert any(fo == 0 for fo, _ in infos)  # calls that gave no output frame
    _, p, infos = stream_path(am, x, [7] * (T // 7) + [T % 7], slot=1, emissions=False)
    assert torch.equal(p, ref_path)
    check_info(tr, infos, ref_path.shape[0])
    am.close()
    tr.close()


@pytest.mark.parametrize("crit,N", [("asg", 30), ("ctc", 30)])
def test_many_streams_match_their_single_stream_path(crit, N):
    """1024 slots, staggered starts, random subsets and chunk lengths per call, and slots restarted while running:
    every stream's joined path is its single-stream path and the Viterbi path of its own emissions"""
    S, Tc = 1024, 24
    tr = make_trainer(crit, N, seed=1)
    am = StreamingAM(tr, S, max_chunk=Tc, precision="f32")
    rng = np.random.default_rng(2)
    lengths = rng.integers(10, 90, S)
    starts = rng.integers(0, 6, S)
    X = features(int(lengths.max()), 3, B=S)
    pos = np.zeros(S, np.int64)
    paths = [[] for _ in range(S)]
    emis = [[] for _ in range(S)]
    state = np.zeros(S, np.int64)  # 0 waiting, 1 running, 2 finished
    restarted = set()
    rnd = 0
    while (state < 2).any():
        new = [s for s in range(S) if state[s] == 0 and starts[s] <= rnd]
        if new:
            am.start(new)
            state[new] = 1
        running = [s for s in range(S) if state[s] == 1]
        # restart a few running slots once: they forget their past and begin again
        again = [s for s in running if pos[s] > 0 and s % 97 == 0 and s not in restarted]
        if again:
            am.start(again)
            restarted.update(again)
            for s in again:
                pos[s], paths[s], emis[s] = 0, [], []
        sub = [s for s in running if rng.random() < 0.8] or running[:1]
        if rnd == 5:
            sub = running  # every stream has started: one round over all of them
        done = [s for s in sub if pos[s] >= lengths[s]]
        go = [s for s in sub if pos[s] < lengths[s]]
        for group, fin in ((go, False), (done, True)):
            if not group:
                continue
            cnt = [int(min(rng.integers(0, Tc + 1), lengths[s] - pos[s])) if not fin else 0 for s in group]
            xc = torch.zeros((len(group), 1, 80, Tc), device="cuda")
            for k, s in enumerate(group):
                xc[k, :, :, :cnt[k]] = X[s, :, :, pos[s]:pos[s] + cnt[k]]
            e, fo, p, info = am.run(group, xc, cnt, finish=fin, path=True)
            info = info.cpu()
            for k, s in enumerate(group):
                emis[s].append(e[k, :fo[k]].clone())
                paths[s].append(p[k, :int(info[k, 1])].clone())
                pos[s] += cnt[k]
            if fin:
                state[group] = 2
        rnd += 1
    single = StreamingAM(tr, 1, max_chunk=Tc, precision="f32")
    for s in range(S):
        e, p = torch.cat(emis[s]), torch.cat(paths[s])
        assert torch.equal(p, viterbi(tr, e)), s
        if s % 61 == 0 or s in restarted:
            x = X[s:s + 1, :, :, :lengths[s]].contiguous()
            _, p1, _ = stream_path(single, x, [Tc] * (int(lengths[s]) // Tc) + [int(lengths[s]) % Tc])
            assert torch.equal(p, p1), s
    single.close()
    am.close()
    tr.close()


@pytest.mark.parametrize("N", [2, 30])
def test_tied_states_force_commits(N):
    """the network's head set to a constant (zero weight, crafted bias), so every output frame is the same emission
    row: states 0 and 1 tie forever and never share a predecessor, and only the pending bound commits frames"""
    tr = make_trainer("asg", N)
    emis_row, trans = tied_forever(N, 1)
    tr.set_flat(torch.from_numpy(trans).reshape(-1).cuda(), which=1)
    flat = tr.get_flat(0).clone()
    w_off, w_n, _ = tr.layout(0)[-2]
    b_off, b_n, _ = tr.layout(0)[-1]
    assert b_n == N
    flat[w_off:w_off + w_n] = 0
    flat[b_off:b_off + b_n] = torch.from_numpy(emis_row[0]).cuda()
    tr.set_flat(flat, which=0)
    chunk = 1000
    am = StreamingAM(tr, 1, max_chunk=chunk, precision="f32")
    model = CarriedViterbi(trans, 1024)
    am.start([0])
    x = features(chunk, 5)
    forced_any = False
    for k in range(12):
        e, fo, p, info = am.run([0], x, path=True)
        rows = e[0, :fo[0]].cpu().numpy()
        assert (rows == emis_row[0]).all()
        labels, first, forced = model.run(rows)
        info = info[0].tolist()
        assert info == [first, len(labels), forced], k
        assert np.array_equal(p[0, :info[1]].cpu().numpy(), labels)
        forced_any |= forced > 0
    e, fo, p, info = am.finish([0], path=True)
    labels, first, forced = model.run(e[0, :fo[0]].cpu().numpy(), finish=True)
    assert info[0].tolist() == [first, len(labels), forced]
    assert np.array_equal(p[0, :len(labels)].cpu().numpy(), labels)
    assert forced_any and model.pending == 0
    am.close()
    tr.close()


@pytest.mark.parametrize("crit", ["ctc", "asg"])
def test_words_of_the_joined_path(crit):
    N = 29 if crit == "ctc" else 28
    tr = make_trainer(crit, N, seed=7)
    text = TextPipeline(LETTERS, "", crit, 0, "" if crit == "ctc" else "|", False, "|")
    am = StreamingAM(tr, 1, max_chunk=64, precision="f32")
    T = 300
    x = features(T, 8)
    e, p, _ = stream_path(am, x, [64] * 4 + [T - 256])
    whole = viterbi(tr, e)
    words = text.ltr2wrd(text.prediction2ltr(p.cpu().numpy()))
    assert words == text.ltr2wrd(text.prediction2ltr(whole.cpu().numpy()))
    assert torch.equal(p, whole)
    text.close()
    am.close()
    tr.close()


def test_bad_arguments_are_refused_before_any_launch():
    tr = make_trainer("asg", 30)
    am = StreamingAM(tr, 2, max_chunk=16, precision="f32")
    am.start([0, 1])
    x = features(16, 1, B=2)
    P = am.max_path_out
    path = torch.empty((2, P), dtype=torch.int32, device="cuda")
    info = torch.empty((2, 3), dtype=torch.int32, device="cuda")
    out = torch.empty(2 * am.max_frames_out * 30, device="cuda")
    fo = (capi.ctypes.c_int * 2)()
    slots = (capi.ctypes.c_int * 2)(0, 1)
    cnt = (capi.ctypes.c_int * 2)(16, 16)
    torch.cuda.synchronize()
    before = capi.launch_count()
    args = (am.h, capi._stream(), 2, slots, cnt, capi._ptr(x), 16, 0, capi._ptr(out), out.numel(), fo)
    rc = capi.lib.w2l_stream_run_path(*args, capi._ptr(path), 2 * P - 1, capi._ptr(info))
    assert rc == 1 and "path buffer too small" in capi.lib.w2l_last_error().decode()
    rc = capi.lib.w2l_stream_run_path(*args, capi._ptr(path), 2 * P, None)
    assert rc == 1
    assert capi.launch_count() == before
    # the slots were not advanced: a good call now gives the fresh-stream result
    rc = capi.lib.w2l_stream_run_path(*args, capi._ptr(path), 2 * P, capi._ptr(info))
    assert rc == 0 and capi.launch_count() > before
    am.close()
    tr.close()
    # ASG over 64 tokens: the emissions stream, the path is refused
    big = make_trainer("asg", 65)
    am = StreamingAM(big, 1, max_chunk=16, precision="f32")
    assert am.max_path_out == 0
    am.start([0])
    e, fo = am.run([0], features(16, 2))
    with pytest.raises(W2LError) as err:
        am.run([0], features(16, 2), path=True)
    assert err.value.code == 4
    am.close()
    big.close()
    # a seq2seq trainer has no streaming model at all
    s2s = Trainer(ARCH, 80, 64, "seq2seq", seq2seq={"hidden": 32, "eos": 62, "pad": 63, "maxdecoderoutputlen": 10})  # encoder out 2H = 64
    with pytest.raises(W2LError, match="seq2seq"):
        StreamingAM(s2s, 1, max_chunk=16)
    s2s.close()


def test_state_bytes_count_the_path():
    ctc, asg = make_trainer("ctc", 30), make_trainer("asg", 30)
    a, b = StreamingAM(ctc, 1, max_chunk=50), StreamingAM(asg, 1, max_chunk=50)
    assert b.state_bytes - a.state_bytes >= 32 * (1024 + b.max_frames_out) + 4 * 32
    for h in (a, b, ctc, asg):
        h.close()
