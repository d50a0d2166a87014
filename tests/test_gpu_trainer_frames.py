"""The trainer's eval-mode entry points on an arch whose explicit padding makes T' larger than Python's first guess of
2T + 64 frames: `PD 0 100 100` before a stride-1 kernel-3 `C2`, as the first stage of archs.streaming_tds() pads its
convolution.  At T = 16, T' = 16 + 200 - 2 = 214.  forward, viterbi_path and align all return those frames, because a
buffer that is too small is refused with t_out already set, and Python calls again at that size.  Each eval entry point
also checks its batch (B, T, features) before it runs anything, and a closed Trainer's NULL handle is refused."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

F, B, T = 80, 2, 16
T_OUT = T + 200 - 2
ARCH = f"V -1 NFEAT 1 0\nPD 0 100 100\nC2 1 4 3 1 1 1 0 0\nR\nRO 2 1 0 3\nV {4 * F} -1 1 0\nL {4 * F} NLABEL\nV NLABEL 0 -1 1\n"
INVALID = 1


def setup():
    from wav2letter_b200.text import TextPipeline
    from wav2letter_b200.trainer import Trainer

    text = TextPipeline("|\n" + "\n".join("abcdefghij") + "\n", "", "ctc", 0, "", False, "|")
    tr = Trainer(ARCH, F, text.num_classes, "ctc", lr=0.0, precision="f32")
    g = torch.Generator(device="cuda").manual_seed(11)
    feat = torch.randn((B, 1, F, T), device="cuda", generator=g)
    target = torch.tensor([[1, 2, 3, 4], [5, 6, -1, -1]], dtype=torch.int32, device="cuda")
    assert 2 * T + 64 < T_OUT
    return text, tr, feat, target


def test_forward_viterbi_path_and_align_return_every_frame():
    _, tr, feat, target = setup()
    N = tr.output_width()
    out = tr.forward(feat)
    assert out.shape == (B, T_OUT, N)
    path = tr.viterbi_path(feat)
    assert path.shape == (B, T_OUT)
    assert torch.equal(path, out.argmax(-1).to(torch.int32))  # CTC's path is the per-frame argmax
    apath, idx = tr.align(feat, target)
    assert apath.shape == idx.shape == (B, T_OUT)
    for b, row in enumerate(apath.cpu().numpy()):  # the forced path spells its target over all T' frames
        labels = [int(v) for k, v in enumerate(row) if v != N - 1 and (k == 0 or v != row[k - 1])]
        assert labels == [int(v) for v in target[b].cpu() if v >= 0], (b, row)


def test_too_small_buffers_report_the_frame_count_and_stay_untouched():
    from wav2letter_b200 import capi

    _, tr, feat, target = setup()
    N = tr.output_width()
    lib, s, fp = capi.lib, capi._stream(), capi._ptr(feat)
    emis = torch.full((B * T_OUT * N,), -7.0, device="cuda")
    path = torch.full((B * T_OUT,), -7, dtype=torch.int32, device="cuda")
    idx = torch.full((B * T_OUT,), -7, dtype=torch.int32, device="cuda")
    calls = {
        "forward_teacher": lambda tout: lib.w2l_trainer_forward_teacher(tr.h, s, B, T, fp, 0, capi._ptr(emis), emis.numel() - 1, tout),
        "viterbi_path": lambda tout: lib.w2l_trainer_viterbi_path(tr.h, s, B, T, fp, None, 0, capi._ptr(path), path.numel() - 1, tout),
        "align": lambda tout: lib.w2l_trainer_align(tr.h, s, B, T, fp, target.shape[1], capi._ptr(target), capi._ptr(path), capi._ptr(idx),
                                                    path.numel() - 1, tout),
    }
    for name, call in calls.items():
        tout = ctypes.c_int(0)
        assert call(ctypes.byref(tout)) == INVALID, name
        assert b"too small" in lib.w2l_last_error(), name
        assert tout.value == T_OUT, name
    torch.cuda.synchronize()
    assert (emis == -7).all() and (path == -7).all() and (idx == -7).all()


def test_eval_entry_points_check_the_batch():
    from wav2letter_b200 import capi
    from wav2letter_b200.trainer import Trainer

    text, tr, feat, target = setup()
    lib, s, fp = capi.lib, capi._stream(), capi._ptr(feat)
    H, maxlen = 32, 10
    s2s = Trainer(f"V -1 NFEAT 1 0\nC2 1 2 5 1 2 1 -1 -1\nR\nV 0 {2 * F} 1 0\nRO 1 0 3 2\nL {2 * F} {2 * H}\n", F, 13, "seq2seq", lr=0.0,
                  seq2seq=dict(hidden=H, eos=11, pad=12, maxdecoderoutputlen=maxlen))
    emis = torch.empty(B * T_OUT * tr.output_width(), device="cuda")
    path = torch.empty(B * T_OUT, dtype=torch.int32, device="cuda")
    idx = torch.empty_like(path)
    loss = torch.empty(B, device="cuda")
    counts = torch.empty((B, 8), dtype=torch.int32, device="cuda")
    tokens = torch.empty(B * 4 * maxlen, dtype=torch.int32, device="cuda")
    lengths = torch.empty(B * 4, dtype=torch.int32, device="cuda")
    scores = torch.empty(B * 4, device="cuda")
    nbest = torch.empty(B, dtype=torch.int32, device="cuda")
    t_out = ctypes.c_int(0)
    tout, p = ctypes.byref(t_out), capi._ptr
    calls = {
        "forward_teacher": lambda b, t, f: lib.w2l_trainer_forward_teacher(tr.h, s, b, t, f, 0, p(emis), emis.numel(), tout),
        "viterbi_path": lambda b, t, f: lib.w2l_trainer_viterbi_path(tr.h, s, b, t, f, None, 0, p(path), path.numel(), tout),
        "align": lambda b, t, f: lib.w2l_trainer_align(tr.h, s, b, t, f, target.shape[1], p(target), p(path), p(idx), path.numel(), tout),
        "evaluate": lambda b, t, f: lib.w2l_trainer_evaluate(tr.h, s, text.to_device(), b, t, f, target.shape[1], p(target), None, None,
                                                             p(loss), p(counts)),
        "decode": lambda b, t, f: lib.w2l_trainer_decode_sized(s2s.h, s, b, t, f, None, p(tokens), p(lengths), tokens.numel()),
        "beam_search": lambda b, t, f: lib.w2l_trainer_beam_search_sized(s2s.h, s, b, t, f, None, 4, maxlen, p(tokens), p(lengths), p(scores),
                                                                         p(nbest), tokens.numel()),
    }
    for name, call in calls.items():
        assert call(B, T, fp) == 0, (name, lib.w2l_last_error())
        for bad in ((0, T, fp), (B, 0, fp), (B, T, None)):
            assert call(*bad) == INVALID, (name, bad)
            assert f"trainer_{name}: bad arguments".encode() in lib.w2l_last_error(), (name, bad, lib.w2l_last_error())


def test_closed_trainer_raises():
    from wav2letter_b200 import W2LError

    _, tr, feat, target = setup()
    tr.close()
    with pytest.raises(W2LError, match="null handle"):
        tr.forward(feat)
    with pytest.raises(W2LError, match="trainer_step_sized: null handle"):
        tr.step(feat, target)
    with pytest.raises(W2LError, match="trainer_viterbi_path: null handle"):
        tr.viterbi_path(feat)
